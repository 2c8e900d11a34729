"""Stages the UNMODIFIED reference packages (linjieli222/HERO: model/ optim/ utils/ data/ config/)
into the git-ignored `oracle/_ref/`, for bench.py's reference arms and the drop-in test. Only the
reference's own .py / .json files are copied, byte for byte; nothing of this project goes there and
nothing under it is tracked or edited. Run by `__graft_entry__.build()`; a machine without a
readable reference checkout simply gets no `oracle/_ref/` (those arms and that test then skip).

    HERO_REFERENCE=<checkout of linjieli222/HERO> python oracle/stage_ref.py
"""
import filecmp
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
PACKAGES = ("model", "optim", "utils", "data", "config")
DEFAULT_REFERENCE = "/root/reference"   # default location of the reference checkout


def available():
    """DEST if a staged copy exists, else None."""
    return DEST if os.path.isfile(os.path.join(DEST, "model", "model.py")) else None


def stage(ref_root=None, verbose=False):
    """Copies the reference packages into DEST; returns available()."""
    ref_root = ref_root or os.environ.get("HERO_REFERENCE") or DEFAULT_REFERENCE
    if not os.access(os.path.join(ref_root, "model", "model.py"), os.R_OK):
        return available()
    for pkg in PACKAGES:
        src, dst = os.path.join(ref_root, pkg), os.path.join(DEST, pkg)
        if not os.path.isdir(src):
            continue
        os.makedirs(dst, exist_ok=True)
        for name in sorted(os.listdir(src)):
            s, d = os.path.join(src, name), os.path.join(dst, name)
            if not os.path.isfile(s) or not name.endswith((".py", ".json")):
                continue
            if not os.path.exists(d) or not filecmp.cmp(s, d, shallow=False):
                shutil.copyfile(s, d)
                if verbose:
                    print("staged", os.path.relpath(d, HERE))
    return available()


if __name__ == "__main__":
    out = stage(sys.argv[1] if len(sys.argv) > 1 else None, verbose=True)
    print("reference staged at", out)
