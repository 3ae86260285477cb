"""Timeline of ONE CUDA-graph replay of the Ape-X learner step (torch.profiler / CUPTI): every kernel with its
stream, start and duration, so the critical path (and what overlaps it) can be read off.
Usage: python tools/prof_timeline.py > timeline.txt"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_rl_b200.apex import ApexConfig, Learner  # noqa: E402

world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
torch.cuda.set_device(dev)
if world > 1:      # torchrun --nproc-per-node N tools/prof_timeline.py: the data-parallel step, rank 0 prints
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
N, B = 1 << 20, 512
cfg = ApexConfig(BATCHSIZE=B, REPLAY_MEMORY_LEN=N, BUFFER_SIZE=0, LEARNER_DEVICE=str(dev))
torch.manual_seed(0)
learner = Learner(cfg, connect=None, start_replay=False)
if world > 1:
    for p in list(learner.model.parameters()) + list(learner.target_model.parameters()):
        dist.broadcast(p.data, 0)
    learner.enable_data_parallel()
st = learner.memory.store
st.fill_hash(N, seed=1 + rank)
st.build((torch.rand(N, device=dev) + 1e-3) ** 0.6)
for _ in range(10):
    learner.fused_step()
torch.cuda.synchronize()
from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(4):
        learner.fused_step()
    torch.cuda.synchronize()
if rank != 0:
    if world > 1:
        dist.barrier()
        learner._graph = None
        dist.destroy_process_group()
    sys.exit(0)
evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
evs.sort(key=lambda e: e.time_range.start)
# split into replays at gaps: take the last replay
starts = [e.time_range.start for e in evs]
n = len(evs) // 4
last = evs[-n:]
t0 = last[0].time_range.start
print(f"# {n} device activities per replay; replay span {last[-1].time_range.end - t0:.1f} us")
streams = {}
for e in last:
    sid = getattr(e, "stream", None)
    if sid is None:
        sid = e.device_index
    streams.setdefault(sid, len(streams))
    print(f"{e.time_range.start - t0:8.1f} {e.time_range.end - t0:8.1f} {e.time_range.end - e.time_range.start:7.1f}  s{streams[sid]:<2d} {e.name[:100]}")
if world > 1:
    dist.barrier()
    learner._graph = None
    dist.destroy_process_group()
