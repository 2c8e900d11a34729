"""Where do the gradient exchanges land on the device timeline of a data-parallel step?
torchrun --nproc-per-node N tools/dp_timeline.py [overlap_ctas]   (rank 0 prints)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile
import bench
from hero_b200 import distributed as hdist, synth
from hero_b200.params import flat_of
from hero_b200.plan import attach_plan

ctas = int(sys.argv[1]) if len(sys.argv) > 1 else 4
rank, world, local = hdist.init()
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
model = bench.build_model(dev)
flat = flat_of(model, dev)
gflat = flat.ensure_flat_grads()
vb, qb = synth.syn_tvr_dense(batch_size=32, seed=1234 + rank)
vbd = synth.to_device(attach_plan(dict(vb)), dev)
qbd = synth.to_device(attach_plan(dict(qb), kind="txt"), dev)
dclip = torch.randn(32, 100, 768, device=dev) * 1e-2
dq = torch.randn(32, 16, 768, device=dev) * 1e-2
bucketer = hdist.GradBucketer(flat)
gflat = flat.ensure_flat_grads()


def step():
    gflat.zero_()
    with bucketer:
        clip, q = model.forward_repr_txt(vbd, qbd)
        torch.autograd.backward([clip, q], [dclip, dq])
    bucketer.finish()


for _ in range(4):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
if rank == 0:
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    t0 = min(e.time_range.start for e in evs)
    t1 = max(e.time_range.end for e in evs)
    print(f"step span {(t1 - t0) / 1e3:.3f} ms, {len(evs)} device activities")
    comp_end = max(e.time_range.end for e in evs if "nccl" not in e.name.lower())
    print(f"last compute kernel ends at {(comp_end - t0) / 1e3:.3f} ms")
    bwd_end = max(e.time_range.end for e in evs if "hero::" in e.name or "gemm_wgmma" in e.name)
    print(f"last hero kernel ends at {(bwd_end - t0) / 1e3:.3f} ms; activities after "
          f"{(bwd_end - t0) / 1e3 - 0.3:.3f} ms:")
    for e in sorted(evs, key=lambda e: e.time_range.start):
        if e.time_range.end > bwd_end - 300 and "nccl" not in e.name.lower():
            print(f"  late  start {(e.time_range.start - t0) / 1e3:7.3f}  end "
                  f"{(e.time_range.end - t0) / 1e3:7.3f}  {e.name[:70]}")
    cp = [e for e in evs if "memcpy" in e.name.lower() and "dtod" in e.name.lower().replace(" ", "")]
    if cp:
        print(f"{len(cp)} DtoD copies: first start {(min(e.time_range.start for e in cp) - t0) / 1e3:.3f}"
              f" last end {(max(e.time_range.end for e in cp) - t0) / 1e3:.3f} ms, total "
              f"{sum(e.time_range.elapsed_us() for e in cp) / 1e3:.3f} ms")
    for e in evs:
        if "nccl" in e.name.lower():
            print(f"  nccl  start {(e.time_range.start - t0) / 1e3:7.3f}  end "
                  f"{(e.time_range.end - t0) / 1e3:7.3f}  dur {e.time_range.elapsed_us() / 1e3:6.3f} ms  "
                  f"{e.name[:60]}")
    # backward start = first ln_bwd / attn bwd kernel
    bw = [e for e in evs if "bwd" in e.name]
    if bw:
        print(f"backward kernels from {(min(e.time_range.start for e in bw) - t0) / 1e3:.3f} ms")
torch.distributed.destroy_process_group()
