"""Per-kernel timings at the BASELINE.json sizes.  Each measurement captures `reps`
launches (distinct inputs) in one CUDA graph and times the replay with CUDA events,
so Python / ctypes launch overhead is excluded.  Diagnostic tool; bench.py is the
judged harness."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_rl_b200 import replay as R  # noqa: E402


def graph_time(fns, iters=5):
    """fns: list of zero-arg callables (one launch group each). -> us per callable (median of iters)."""
    for f in fns[:2]:
        f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for f in fns:
            f()
    g.replay(); torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); g.replay(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3 / len(fns))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--payload", type=int, default=1)
    ap.add_argument("--tag", default="")
    ap.add_argument("--out", default=".", help="directory for microbench<tag>.json")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    N = 1 << args.log2n
    rep = R.DeviceReplay(N, fields=R.APEX_FIELDS if args.payload else (), device=dev)
    if args.payload:
        rep.fill_hash(N)
    p = (torch.randn(N, device=dev).abs().clamp(max=1) + 1e-7) ** 0.6
    rep.build(p)
    res = {"N": N, "gather_mode": os.environ.get("B2RL_GATHER", "bulk"), "update_mode": os.environ.get("B2RL_UPDATE", "auto")}
    res["build_us"] = graph_time([lambda: rep.build(p)] * 4)
    res["build_GBs_8N"] = 8 * N / res["build_us"] / 1e3
    reps = 10
    for n in (512, 4096, 8192, 65536):
        outs = [(torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev))
                for _ in range(reps)]
        res[f"sample_{n}_us"] = t = graph_time([(lambda o=o: rep.sample(n, out=o)) for o in outs])
        res[f"sample_{n}_GBs_88B"] = 88 * n / t / 1e3
        vals = torch.rand(n, device=dev) + 0.01
        res[f"update_{n}_us"] = t = graph_time([(lambda o=o: rep.update(o[0], vals)) for o in outs])
        res[f"update_{n}_GBs_164B"] = 164 * n / t / 1e3
        if args.payload and n <= 8192:
            ob = rep.alloc_batch(n)
            res[f"gather_{n}_us"] = t = graph_time([(lambda o=o: rep.gather(o[0], ob)) for o in outs])
            res[f"gather_{n}_GBs_alg"] = 56457 * n / t / 1e3
    B, A = 512, 6
    q = [torch.randn(B, A, device=dev) for _ in range(3)]
    a = torch.randint(0, A, (B,), device=dev); r = torch.randn(B, device=dev)
    nd = torch.ones(B, device=dev); w = torch.rand(B, device=dev)
    out = R.apex_target(*q, a, r, nd, w, 0.97, 0.6)
    res["apex_target_512_us"] = graph_time([lambda: R.apex_target(*q, a, r, nd, w, 0.97, 0.6, out=out)] * 10)
    if args.payload:
        wt = torch.empty(32, 4, 8, 8, device=dev).uniform_(-0.06, 0.06)
        for nn_ in (1, 2):
            pack = R.Conv1Pack(nn_, dev)
            for i in range(nn_):
                pack.pack(i, wt)
            field = rep.field_view("next_state")
            for n in (512, 4096):
                idxs = [rep.sample(n)[0] for _ in range(6)]
                out = torch.empty((nn_, n, 20, 20, 32), device=dev)
                t = graph_time([(lambda ix=ix: R.conv1_fused(field, ix, pack, relu=True, out=out)) for ix in idxs])
                res[f"conv1_fused_{nn_}net_{n}_us"] = t
                res[f"conv1_fused_{nn_}net_{n}_frames_GBs"] = 28224 * n / t / 1e3
                res[f"conv1_fused_{nn_}net_{n}_TOPS_i8"] = 2.0 * 512 * (128 * nn_) * 256 * n / t / 1e6
        res["conv1_pack_us"] = graph_time([lambda: pack.pack(0, wt)] * 10)
    print(json.dumps(res, indent=1))
    os.makedirs(args.out, exist_ok=True)
    json.dump(res, open(os.path.join(args.out, f"microbench{args.tag}.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
