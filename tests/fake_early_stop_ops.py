"""TEST INFRASTRUCTURE: torch restatement of the TVC early-stop entry point (include/hero_b200.h:
hero_dec_finished), in the style of tests/fake_decode_ctl_ops.py, so early stop runs on a CPU-only
box. Also used on the GPU as the restatement the kernel is checked against.

The rule, as csrc/decode_ctl.cu states it: with ids, fin[r] |= (ids[r] == eos) for r < rows;
without, fin is only read. If every fin[r] is set (rows == 0 included) and stop_dev still holds
INT32_MAX, stop_dev = step and the host word stop_host = step; otherwise nothing changes. Here the
host word is written directly. It must be a host tensor, pinned whenever the flags live on a GPU
(where the kernel writes it through its device mapping).
"""
import torch


def dec_finished(ids, fin, stop_dev, stop_host, *, rows, eos, step):
    if int(rows) != rows or rows < 0 or int(step) != step or step < 0:
        raise ValueError(f"dec_finished: rows {rows}, step {step}")
    if not isinstance(stop_host, torch.Tensor) or stop_host.is_cuda \
            or stop_host.dtype != torch.int32 or stop_host.numel() < 1 \
            or (fin.is_cuda and not stop_host.is_pinned()):
        raise ValueError("dec_finished: stop_host must be an int32 tensor in pinned host memory")
    if fin.numel() < rows or (ids is not None and ids.numel() < rows):
        raise ValueError(f"dec_finished: {rows} rows")
    f = fin.view(-1)[:rows]
    if ids is not None:
        f |= (ids.view(-1)[:rows] == eos).to(f.dtype)
    from hero_b200 import ops
    if bool((f != 0).all()) and int(stop_dev.view(-1)[0]) == ops.DEC_STOP_UNSET:
        stop_dev.view(-1)[0] = step
        stop_host.view(-1)[0] = step


def install(monkeypatch):
    from tests import fake_decode_ctl_ops
    fake_decode_ctl_ops.install(monkeypatch)
    from hero_b200 import ops
    monkeypatch.setattr(ops, "dec_finished", dec_finished)
