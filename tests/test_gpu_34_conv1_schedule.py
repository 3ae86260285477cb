"""GPU tests of conv_1's work split (csrc/conv1.cu, csrc/conv1_wgrad.cu): batch sizes that give a CTA one stack, a
single tile or the last tile's empty upper half alone, stacks whose tiles are split across CTAs, fewer stacks than SMs,
counts that are not a multiple of the SM count, and more items per CTA than the weight gradient keeps ReLU masks on chip
for, held to the fp64 bounds of tests/fp64_bounds.py; then every frame kind bit for bit against frame stacks holding
the same pixels at the same batch sizes."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from apex_atari_records import atari_records              # noqa: E402
from fp64_bounds import check_conv1, check_wgrad          # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_rl_b200 import replay
    return replay


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes():
    s = _sms()
    # 1: four CTAs of one tile each, the last one the empty upper half's tile; s // 4 + 1: every CTA a tile or two of
    # a stack split across CTAs; s - 1, s + 1, 2 s + 3: one stack per CTA give or take, units not a multiple of the grid;
    # 5 s + 7: more items per CTA than the weight gradient keeps ReLU masks on chip for (it reads y again for the rest)
    return sorted({1, 2, s // 4 + 1, s - 1, s + 1, 2 * s + 3, 5 * s + 7})


def _packs(R, c_out, g):
    ws = [torch.randn(c_out, 4, 8, 8, device="cuda", generator=g) * 0.05 for _ in range(2)]
    packs = {}
    for n_nets in (1, 2):
        packs[n_nets] = R.Conv1Pack(n_nets, "cuda", c_out)
        for k in range(n_nets):
            packs[n_nets].pack(k, ws[k])
    return ws, packs


@pytest.mark.parametrize("c_out", [32, 16])
def test_schedule_edge_cases_against_fp64(R, c_out):
    g = torch.Generator(device="cuda").manual_seed(34)
    ws, packs = _packs(R, c_out, g)
    frames = torch.randint(0, 256, (600, 4, 84, 84), dtype=torch.uint8, device="cuda", generator=g)
    for n in _sizes():
        idx = torch.randint(0, 600, (n,), device="cuda", generator=g)
        for n_nets in (1, 2):
            for relu in (True, False):
                outs = R.conv1_fused(frames, idx, packs[n_nets], relu=relu)
                check_conv1(f"conv1 n={n} nets={n_nets} relu={relu}", frames, idx, ws[:n_nets], outs, relu)
                if n_nets == 2:   # each network of a two-network launch equals its one-network launch
                    assert torch.equal(outs[0], R.conv1_fused(frames, idx, packs[1], relu=relu)[0])
        y = R.conv1_fused(frames, idx, packs[1], relu=True)[0]
        gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
        for relu_y in (y, None):
            gw = R.conv1_wgrad(frames, idx, gy, relu_y=relu_y)
            check_wgrad(f"wgrad n={n} masked={relu_y is not None}", frames, idx, gy, gw, relu_y=relu_y)


def _coded_store(R):
    cap, F, W = 1024, 4096, 256
    st = R.CodedDedupReplay(cap, F, W, 16 * (W + 2 + 8 * 40) * 442)
    s, ns, a, r, d = atari_records(700, actors=9, seed=5)
    p = np.random.default_rng(105).random(700).astype(np.float32) + 0.01
    for i in range(0, 700, 100):
        sl = slice(i, i + 100)
        st.push([torch.from_numpy(x[sl]) for x in (s, ns, a, r, d)], torch.from_numpy(p[sl]))
    torch.cuda.synchronize()
    return st


@pytest.mark.parametrize("c_out", [32, 16])
def test_every_frame_kind_equals_frame_stacks(R, c_out):
    g = torch.Generator(device="cuda").manual_seed(35)
    _, packs = _packs(R, c_out, g)
    flat = torch.randint(0, 256, ((500 + 3) * 7056,), dtype=torch.uint8, device="cuda", generator=g)
    strips = torch.as_strided(flat, (500, 4, 84, 84), (7056, 7056, 84, 1))          # overlapping 4-frame windows
    pool = torch.randint(0, 256, (900, 84, 84), dtype=torch.uint8, device="cuda", generator=g)
    planes = torch.randint(0, 900, (500, 8), dtype=torch.int32, device="cuda", generator=g)
    coded = _coded_store(R)
    # (source, rows, the same rows as frame stacks)
    kinds = {"strips": (strips, 500, strips.contiguous()),
             "planes": (R.PlaneFrames(pool, planes, 4, 8), 500, pool[planes[:, 4:].long()]),
             "coded": (coded.frame_source("next_state"), 700, coded.gather(torch.arange(700, device="cuda"))["next_state"])}
    for name, (src, rows, stacks) in kinds.items():
        for n in _sizes():
            idx = torch.randint(0, rows, (n,), device="cuda", generator=g)
            for n_nets in (1, 2):
                for u, v in zip(R.conv1_fused(src, idx, packs[n_nets], relu=True),
                                R.conv1_fused(stacks, idx, packs[n_nets], relu=True)):
                    assert torch.equal(u, v), (name, n, n_nets)
            y = R.conv1_fused(stacks, idx, packs[1], relu=True)[0]
            gy = torch.randn(n, c_out, 20, 20, device="cuda", generator=g)
            assert torch.equal(R.conv1_wgrad(src, idx, gy, relu_y=y), R.conv1_wgrad(stacks, idx, gy, relu_y=y)), (name, n)
