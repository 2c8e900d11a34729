"""Stages the reference's UNMODIFIED pure-Python COCO caption scorers (eval/pycocoevalcap/
__init__.py, bleu/, cider/, rouge/) into the git-ignored `oracle/_ref/eval/`, beside the packages
oracle/stage_ref.py stages, for the reference arm of tools/caption_metrics_probe.py. Only the
reference's own .py files are copied, byte for byte; nothing Java-based (tokenizer/, meteor/) is.
Run by `__graft_entry__.build()`; without a readable reference checkout nothing is staged.

    HERO_REFERENCE=<checkout of linjieli222/HERO> python oracle/stage_caption_scorers.py
"""
import filecmp
import os
import shutil
import sys

try:
    from .stage_ref import DEFAULT_REFERENCE, DEST
except ImportError:                    # run as a script
    from stage_ref import DEFAULT_REFERENCE, DEST

SCORERS = ("eval/pycocoevalcap", "eval/pycocoevalcap/bleu", "eval/pycocoevalcap/cider",
           "eval/pycocoevalcap/rouge")


def available():
    """The directory to put on sys.path for `import pycocoevalcap` if it is staged, else None."""
    root = os.path.join(DEST, "eval")
    return root if os.path.isfile(os.path.join(root, "pycocoevalcap", "cider", "cider.py")) \
        else None


def stage(ref_root=None, verbose=False):
    """Copies the scorers into DEST/eval; returns available()."""
    ref_root = ref_root or os.environ.get("HERO_REFERENCE") or DEFAULT_REFERENCE
    if not os.access(os.path.join(ref_root, "eval", "pycocoevalcap", "__init__.py"), os.R_OK):
        return available()
    for pkg in SCORERS:
        src, dst = os.path.join(ref_root, pkg), os.path.join(DEST, pkg)
        if not os.path.isdir(src):
            continue
        os.makedirs(dst, exist_ok=True)
        for name in sorted(os.listdir(src)):
            s, d = os.path.join(src, name), os.path.join(dst, name)
            if not os.path.isfile(s) or not name.endswith(".py"):
                continue
            if not os.path.exists(d) or not filecmp.cmp(s, d, shallow=False):
                shutil.copyfile(s, d)
                if verbose:
                    print("staged", os.path.relpath(d, os.path.dirname(DEST)))
    return available()


if __name__ == "__main__":
    out = stage(sys.argv[1] if len(sys.argv) > 1 else None, verbose=True)
    print("caption scorers staged at", out)
