"""GraphAgent — the Q / policy network the targets are computed from.

The reference describes its networks as a JSON graph of named nodes executed in
`prior` order (baseline/baseAgent.py:60-180, 287-309; layer zoo in
baseline/baseNetwork.py).  The network is a *callee* of the hot path and stays
plain PyTorch (SURVEY.md §2 row 10, §8f rank 2); this module is an independent,
much smaller interpreter for the node types the three shipped configs use
(cfg/ape_x.json, cfg/r2d2.json, cfg/impala.json):

    CNN2D  MLP  LSTMNET  ViewV2  Add  Mean  Substract

and RESCNN2D, the IMPALA paper's residual network (impala.resnet_small_model, and r2d2.resnet_model in front of
R2D2's LSTM; no shipped config uses it, a config selects it through its MODEL dict), with the same call surface the
learners rely on: forward([inputs]) -> tuple,
getParameters, updateParameter(other, tau), setCellState / detachCellState /
zeroCellState, calculateNorm, clippingNorm, and state_dict() key names
(`module00.conv_1.weight`, `module02.MLP_1.weight`, `module02.rnn.weight_ih_l0`,
...) so that reference actors can load the weights this learner publishes.
All layers are bias-free, as in the reference (baseNetwork.py:77-79,165-172).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn as nn

_ACT = {"relu": nn.ReLU, "tanh": nn.Tanh, "sigmoid": nn.Sigmoid, "linear": None}


def _act(name):
    if name not in _ACT:
        raise ValueError(f"unsupported activation {name!r}")
    return None if _ACT[name] is None else _ACT[name]()


class _ConvSplitBackward(torch.autograd.Function):
    """conv2d whose backward computes dL/dx on the current stream and hands dL/dW to the active
    WeightGradSink (linear.py): the weight gradient only feeds the optimizer, so it leaves the critical path."""

    @staticmethod
    def forward(ctx, x, w, stride, padding):
        from .linear import taped
        ctx.save_for_backward(x, w)
        ctx.sp = (tuple(stride), tuple(padding))
        return taped(lambda: torch.nn.functional.conv2d(x, w, None, stride, padding))

    @staticmethod
    def backward(ctx, gy):
        from . import linear as _lin
        WeightGradSink = _lin.WeightGradSink
        x, w = ctx.saved_tensors
        stride, padding = ctx.sp
        bw = torch.ops.aten.convolution_backward

        def run(mask):
            return bw(gy, x, w, None, stride, padding, (1, 1), False, (0, 0), 1, mask)

        # the weight gradient is handed to the sink BEFORE dL/dx is launched: its lane forks from the stream as it is
        # now (gy complete) and runs beside this layer's own dgrad instead of behind it
        gw = None
        if ctx.needs_input_grad[1]:
            if WeightGradSink.usable((w,)):
                sink = _lin._SINK
                sink.submit(lambda: sink.accumulate(w, run((False, True, False))[1]), keep=(gy, x), lane=1)
            else:
                gw = run((False, True, False))[1]
        gx = run((True, False, False))[0] if ctx.needs_input_grad[0] else None
        return gx, gw, None, None


class ConvStack(nn.Sequential):
    """netCat CNN2D: conv layers (bias=False), then Flatten at fSize == -1."""

    def __init__(self, d):
        super().__init__()
        ch = d["iSize"]
        acts = list(d["act"]) if isinstance(d["act"], list) else [d["act"]] * d["nLayer"]
        for i, k in enumerate(d["fSize"]):
            if k == -1:
                self.add_module("Flatten", nn.Flatten())
                continue
            self.add_module(f"conv_{i + 1}", nn.Conv2d(ch, d["nUnit"][i], k, stride=d["stride"][i],
                                                       padding=d["padding"][i], bias=False))
            ch = d["nUnit"][i]
            a = _act(acts[i]) if i < len(acts) else None
            if a is not None:
                self.add_module(f"act_{i + 1}", a)

    split_backward = False     # route Conv2d layers through _ConvSplitBackward (set by the learner)

    def _run(self, layer, x):
        from . import linear as _lin
        taping = _lin._TAPE is not None
        if (self.split_backward or taping) and isinstance(layer, nn.Conv2d) and x.is_cuda \
                and (torch.is_grad_enabled() or taping) \
                and layer.bias is None and layer.dilation == (1, 1) and layer.groups == 1:
            return _ConvSplitBackward.apply(x, layer.weight, layer.stride, layer.padding)
        if taping and isinstance(layer, nn.ReLU):
            return _lin._ReluTaped.apply(x)
        return layer(x)

    def forward(self, xs):
        x = xs[0] if isinstance(xs, (tuple, list)) else xs
        for layer in self:
            x = self._run(layer, x)
        return x

    def is_atari_conv1(self) -> bool:
        """True if the first layer is the 8x8/stride-4, 4->32 (or 4->16), bias-free conv followed by ReLU
        that libb2rl's fused gather+conv1 kernel implements (cfg/ape_x.json, cfg/r2d2.json, cfg/impala.json)."""
        layers = list(self.children())
        if len(layers) < 2 or not isinstance(layers[0], nn.Conv2d) or not isinstance(layers[1], nn.ReLU):
            return False
        c = layers[0]
        return (c.in_channels, c.kernel_size, c.stride, c.padding, c.bias) == (4, (8, 8), (4, 4), (0, 0), None) \
            and c.out_channels in (16, 32)

    def forward_tail(self, y, relu_applied: bool, stop_before_head: bool = False):
        """Continue after conv_1: `y` is conv_1's output (pre- or post-ReLU).  stop_before_head: return the LAST
        conv's pre-ReLU output instead of running the closing ReLU + Flatten (ends_with_relu_flatten() must hold):
        linear.relu_flat_linear3x folds those two into the heads' operand packing."""
        layers = list(self.children())[2 if relu_applied else 1:]
        if stop_before_head:
            layers = layers[:-2]
        x = y
        for layer in layers:
            x = self._run(layer, x)
        return x

    def ends_with_relu_flatten(self) -> bool:
        layers = list(self.children())
        return (len(layers) >= 4 and isinstance(layers[-3], nn.Conv2d) and isinstance(layers[-2], nn.ReLU)
                and isinstance(layers[-1], nn.Flatten))


class ResidualBlock(nn.Module):
    """x + conv_2(relu(conv_1(relu(x)))), both convs 3x3 / stride 1 / pad 1, bias-free."""

    def __init__(self, ch):
        super().__init__()
        self.act_1 = nn.ReLU()
        self.conv_1 = nn.Conv2d(ch, ch, 3, stride=1, padding=1, bias=False)
        self.act_2 = nn.ReLU()
        self.conv_2 = nn.Conv2d(ch, ch, 3, stride=1, padding=1, bias=False)

    def forward(self, x):
        return x + self.conv_2(self.act_2(self.conv_1(self.act_1(x))))


class ResidualStack(nn.Sequential):
    """netCat RESCNN2D: the IMPALA paper's "large" network without its LSTM (Espeholt et al. 2018, Fig. 3).  Section
    i = 1..len(nUnit) is conv_i (3x3, stride 1, pad 1), pool_i (3x3 max-pool, stride 2, pad 1) and blockNum residual
    blocks block_i_j; then a ReLU and, with `linear`, a Flatten.  Every conv is bias-free.  84x84 frames give 42, 21
    and 11: 32 * 11 * 11 = 3 872 features at nUnit [16, 32, 32].  The first conv and pool are the stem libb2rl runs
    fused with the frame gather (csrc/stem.cu)."""

    def __init__(self, d):
        super().__init__()
        ch = d["iSize"]
        for i, c in enumerate(d["nUnit"], 1):
            self.add_module(f"conv_{i}", nn.Conv2d(ch, c, 3, stride=1, padding=1, bias=False))
            self.add_module(f"pool_{i}", nn.MaxPool2d(3, stride=2, padding=1))
            for j in range(1, d["blockNum"] + 1):
                self.add_module(f"block_{i}_{j}", ResidualBlock(c))
            ch = c
        self.add_module("act", nn.ReLU())
        if d.get("linear", True):
            self.add_module("Flatten", nn.Flatten())

    def forward(self, xs):
        x = xs[0] if isinstance(xs, (tuple, list)) else xs
        for layer in self:
            x = layer(x)
        return x

    def is_fused_stem(self) -> bool:
        """True if the stem is the 3x3 / stride-1 / pad-1, 4 -> 16 channel conv that libb2rl's stem kernels run."""
        c = self.conv_1
        return (c.in_channels, c.out_channels, c.kernel_size, c.stride, c.padding) == (4, 16, (3, 3), (1, 1), (1, 1))

    def forward_tail(self, p):
        """Continue after the stem: `p` is pool_1's output."""
        x = p
        for layer in list(self.children())[2:]:
            x = layer(x)
        return x


class DenseStack(nn.Sequential):
    """netCat MLP: Linear layers (bias off unless cfg says so) with activations."""

    def __init__(self, d):
        super().__init__()
        n_in = d["iSize"]
        acts = d["act"] if isinstance(d["act"], list) else [d["act"]] * d["nLayer"]
        bias = bool(d.get("bias", False))
        for i in range(d["nLayer"]):
            self.add_module(f"MLP_{i + 1}", nn.Linear(n_in, d["fSize"][i], bias=bias))
            n_in = d["fSize"][i]
            a = _act(acts[i])
            if a is not None:
                self.add_module(f"act_{i + 1}", a)

    dense_3xtf32 = False      # bias-free wide layers through linear.linear3x (set by GraphAgent / the learner)

    def _layer(self, layer, x):
        if (self.dense_3xtf32 and isinstance(layer, nn.Linear) and layer.bias is None and x.is_cuda and x.dim() == 2
                and x.dtype == torch.float32 and layer.out_features >= 64 and layer.in_features >= 64):
            from .linear import linear3x          # fp32 SIMT sgemm -> 3xTF32 wgmma GEMM at fp32 accuracy
            return linear3x(x, layer.weight)
        return layer(x)

    def forward(self, xs):
        x = xs[0] if isinstance(xs, (tuple, list)) else xs
        for layer in self:
            x = self._layer(layer, x)
        return x

    def forward_after_first(self, h):
        """Continue after the first Linear (its output `h` was computed jointly with sibling heads)."""
        x = h
        for layer in list(self.children())[1:]:
            x = layer(x)
        return x


class Recurrent(nn.Module):
    """netCat LSTMNET: single-layer LSTM that carries its cell state between calls."""

    def __init__(self, d):
        super().__init__()
        self.hidden = d["hiddenSize"]
        self.flatten = bool(d.get("FlattenMode", False))
        self.return_hidden = bool(d.get("return_hidden", False))
        self.rnn = nn.LSTM(d["iSize"], self.hidden, d.get("nLayer", 1))
        self.state = None

    def set_state(self, hc):
        self.state = hc

    def detach_state(self):
        if self.state is not None:
            self.state = (self.state[0].detach().clone(), self.state[1].detach().clone())

    def zero_state(self, num=1):
        p = next(self.rnn.parameters())
        z = torch.zeros(1, num, self.hidden, device=p.device, dtype=p.dtype)
        self.state = (z, z.clone())

    def forward(self, xs):
        x = xs[0]
        if self.state is None:
            self.zero_state(x.shape[1])
        out, hc = self.rnn(x, self.state)
        self.state = hc
        if self.return_hidden:
            return out[-1:]
        if self.flatten:
            out = out.reshape(-1, self.hidden)
        return out


class ViewAs(nn.Module):
    """netCat ViewV2: inputs = (shape tensor, activations) -> activations.view(shape)."""

    def forward(self, xs):
        shape, x = xs[0], xs[1]
        dims = tuple(int(v) for v in (shape.tolist() if torch.is_tensor(shape) else shape))
        return x.view(dims)


class _PreHead:
    """Marker for a conv stack's output that has NOT been through its closing ReLU + Flatten yet."""

    def __init__(self, y):
        self.y = y


class _Add(nn.Module):
    def forward(self, xs):
        return xs[0] + xs[1]


class _Sub(nn.Module):
    def forward(self, xs):
        return xs[0] - xs[1]


class _Mean(nn.Module):
    def forward(self, xs):
        return xs[0].mean(dim=-1, keepdim=True)


def _refresh_after_load(module, incompatible_keys):
    module.refresh_resident_heads()


_NODE = {"CNN2D": ConvStack, "RESCNN2D": ResidualStack, "MLP": DenseStack, "LSTMNET": Recurrent,
         "ViewV2": lambda d: ViewAs(), "Add": lambda d: _Add(), "Substract": lambda d: _Sub(),
         "Mean": lambda d: _Mean()}


class GraphAgent(nn.Module):
    def __init__(self, model_cfg: dict):
        super().__init__()
        self.cfg = model_cfg
        order = sorted(model_cfg, key=lambda n: (model_cfg[n]["prior"], n))
        self._order = order
        self._ext = {}      # node -> list of external input ids
        self._prev = {}     # node -> list of upstream node names
        self._outputs = [n for n in sorted(model_cfg) if model_cfg[n].get("output")]
        self._recurrent = []
        for name in order:
            d = model_cfg[name]
            kind = d["netCat"]
            if kind not in _NODE:
                raise ValueError(f"node type {kind!r} is not used by the shipped configs and is not supported")
            setattr(self, name, _NODE[kind](d))
            self._ext[name] = list(d.get("input", []))
            self._prev[name] = list(d.get("prevNodeNames", []))
            if kind == "LSTMNET":
                self._recurrent.append(name)
        # Sibling MLP heads fed by the same node (the dueling adv/val heads): their first Linear layers
        # share the input, so they run as ONE GEMM on the concatenated weights (same maths, wider N).
        self.fuse_sibling_heads = True
        self.dense_3xtf32 = False       # first Linear of fused sibling heads via linear.linear3x (csrc/gemm.cu)
        self._pack_cache = None         # see packed_heads_cache()
        # Persistent operand images of the fused heads' first layers ({group: {"fwd", "bwdT"?}}), see
        # keep_resident_heads().  RULE: every write of those weights must leave the images equal to packing the new
        # weights.  The fused optimizer does it in the update itself (FusedRMSprop.write_images); updateParameter and
        # load_state_dict repack them (refresh_resident_heads); any other in-place write must call that too.
        self._resident = None
        self.register_load_state_dict_post_hook(_refresh_after_load)
        groups = {}
        for name in order:
            m = getattr(self, name)
            if isinstance(m, DenseStack) and not self._ext[name] and len(self._prev[name]) == 1:
                first = next(iter(m.children()))
                if isinstance(first, nn.Linear) and first.bias is None:
                    groups.setdefault((self._prev[name][0], first.in_features), []).append(name)
        self._head_groups = {n: tuple(g) for g in groups.values() if len(g) > 1 for n in g}
        # Dueling tail: two 2-layer heads (relu, linear) combined by Add / Mean / Substract nodes
        # (cfg/ape_x.json:52-88) -> one kernel after the shared first layer (csrc/dueling.cu).
        self.fused_dueling_tail = False
        self.fused_relu_flatten = True      # act_3 + Flatten folded into the heads' operand packs (linear._ReluFlatLinear3x)
        self._dueling = {}
        for g in set(self._head_groups.values()):
            d = self._match_dueling(g)
            if d is not None:
                self._dueling[g] = d

    def _match_dueling(self, group):
        if len(group) != 2:
            return None
        cfg = self.cfg

        def two_layer(name):
            layers = list(getattr(self, name).children())
            return (len(layers) == 3 and isinstance(layers[0], nn.Linear) and isinstance(layers[1], nn.ReLU)
                    and isinstance(layers[2], nn.Linear) and layers[0].bias is None and layers[2].bias is None)

        if not all(two_layer(n) for n in group):
            return None
        users = {n: [m for m in self._order if n in self._prev[m]] for n in self._order}
        for adv, val in (group, group[::-1]):
            if getattr(self, val).MLP_2.out_features != 1 or \
                    getattr(self, adv).MLP_1.out_features != getattr(self, val).MLP_1.out_features:
                continue
            mean = [m for m in users[adv] if cfg[m]["netCat"] == "Mean" and self._prev[m] == [adv]]
            add = [m for m in users[adv] if cfg[m]["netCat"] == "Add" and sorted(self._prev[m]) == sorted([adv, val])]
            if len(mean) != 1 or len(add) != 1:
                continue
            sub = [m for m in users[add[0]] if cfg[m]["netCat"] == "Substract" and self._prev[m] == [add[0], mean[0]]]
            inner = (adv, val, add[0], mean[0])
            if len(sub) != 1 or sorted(users[adv]) != sorted([mean[0], add[0]]) or users[val] != [add[0]] \
                    or users[add[0]] != sub or users[mean[0]] != sub or any(n in self._outputs for n in inner):
                continue
            return {"adv": adv, "val": val, "inner": inner, "out": sub[0]}
        return None

    # -- execution: external inputs first, then upstream outputs (reference order) --
    def forward(self, inputs, preset: dict | None = None):
        """`preset` maps node names to already-computed outputs (used by the fused conv_1 path)."""
        vals = dict(preset) if preset else {}
        first_out = {}
        for name in self._order:
            if name in vals:
                continue
            group = self._head_groups.get(name) if self.fuse_sibling_heads else None
            if group is not None:
                duel = self._dueling.get(group) if self.fused_dueling_tail else None
                if duel is not None and name not in first_out:
                    from .linear import dueling_tail, dueling_tail_supported, linear3x
                    x = vals[self._prev[name][0]]
                    adv, val = getattr(self, duel["adv"]), getattr(self, duel["val"])
                    pre = x if isinstance(x, _PreHead) else None
                    if pre is not None:
                        from .linear import relu_flat_heads_dueling
                        ws = [adv.MLP_1.weight, val.MLP_1.weight]
                        cache = None if self._pack_cache is None else self._pack_cache.setdefault(group, {})
                        vals[duel["out"]] = relu_flat_heads_dueling(pre.y, ws, adv.MLP_2.weight, val.MLP_2.weight, cache)
                        for n in duel["inner"]:
                            vals[n] = None
                        continue
                    if x.is_cuda and x.dim() == 2 and x.dtype == torch.float32:
                        ws = [adv.MLP_1.weight, val.MLP_1.weight]
                        if self.dense_3xtf32:
                            cache = None if self._pack_cache is None else self._pack_cache.setdefault(group, {})
                            h = linear3x(x, ws, cache)
                        else:
                            h = torch.nn.functional.linear(x, torch.cat(ws, 0))
                        if dueling_tail_supported(h, adv.MLP_2.weight, val.MLP_2.weight):
                            vals[duel["out"]] = dueling_tail(h, adv.MLP_2.weight, val.MLP_2.weight)
                            for n in duel["inner"]:
                                vals[n] = None
                            continue
                        for n, part in zip((duel["adv"], duel["val"]), torch.split(h, [w.shape[0] for w in ws], dim=-1)):
                            first_out[n] = part
                if name not in first_out:
                    x = vals[self._prev[name][0]]
                    ws = [next(iter(getattr(self, n).children())).weight for n in group]
                    if self.dense_3xtf32 and x.is_cuda and x.dim() == 2 and x.dtype == torch.float32:
                        from .linear import linear3x
                        cache = None if self._pack_cache is None else self._pack_cache.setdefault(group, {})
                        h = linear3x(x, ws, cache)
                    else:
                        h = torch.nn.functional.linear(x, torch.cat(ws, 0))
                    for n, part in zip(group, torch.split(h, [w.shape[0] for w in ws], dim=-1)):
                        first_out[n] = part
                vals[name] = getattr(self, name).forward_after_first(first_out[name])
                continue
            srcs = [inputs[i] for i in self._ext[name]] + [vals[p] for p in self._prev[name]]
            node = getattr(self, name)
            if isinstance(node, DenseStack):
                node.dense_3xtf32 = self.dense_3xtf32
            vals[name] = node(tuple(srcs))
        return tuple(vals[n] for n in self._outputs)

    @contextlib.contextmanager
    def packed_heads_cache(self, packs: dict | None = None):
        """While active, the packed (3xTF32) forward operand of the fused heads is built once and reused by
        every forward pass: use it around several passes between which the weights do not change.  `packs`:
        operands prepack_heads() already built for these weights (e.g. on another stream), used from the start."""
        self._pack_cache = dict(packs) if packs else {}
        try:
            yield
        finally:
            self._pack_cache = None

    def prepack_heads(self, transposed: bool = False) -> dict:
        """Fill the packed-operand cache (inside packed_heads_cache()) without running a forward pass, so
        that passes issued on several streams afterwards only read it.  transposed=True prepares the W^T
        operand the input-gradient GEMM of a later backward pass needs (entry "bwdT").  Returns the cache
        entries it filled, which packed_heads_cache(packs) accepts."""
        built = {}
        if self._pack_cache is None:
            return built
        from .linear import _pack_pieces
        for group, ws in self.head_pieces():
            entry = built[group] = self._pack_cache.setdefault(group, {})
            entry["bwdT" if transposed else "fwd"] = _pack_pieces(ws, transposed, True)
        return built

    def head_pieces(self):
        """[(group, first-layer weights in operand order)] of the sibling head groups the 3xTF32 GEMM runs fused."""
        if not (self.dense_3xtf32 and self.fuse_sibling_heads):
            return []
        out = []
        for group in sorted(set(self._head_groups.values())):
            duel = self._dueling.get(group) if self.fused_dueling_tail else None
            names = (duel["adv"], duel["val"]) if duel is not None else group
            ws = [next(iter(getattr(self, n).children())).weight for n in names]
            if ws[0].is_cuda and not any(w.shape[0] % 32 for w in ws[:-1]):
                out.append((group, ws))
        return out

    def keep_resident_heads(self, transposed: bool) -> dict:
        """Allocate and pack persistent operand images of the fused heads: "fwd" (and "bwdT", the W^T operand of
        dL/dx, if `transposed`) per group, in the form packed_heads_cache(packs) takes.  See the rule in __init__."""
        from .linear import _pack_pieces
        self._resident = {group: {k: _pack_pieces(ws, k == "bwdT", True) for k in (("fwd", "bwdT") if transposed
                                                                                else ("fwd",))}
                          for group, ws in self.head_pieces()}
        return self._resident

    def refresh_resident_heads(self) -> None:
        """Repack the resident images (in place: captured graphs keep reading them) from the current weights."""
        if not self._resident:
            return
        from .linear import _pack_pieces
        for group, ws in self.head_pieces():
            for k, img in self._resident[group].items():
                _pack_pieces(ws, k == "bwdT", True, out=img)

    def _prehead_group(self):
        """(group, (C, HW)) if the first conv node ends with [Conv2d, ReLU, Flatten] and feeds ONLY one dueling head
        group that runs on the 3xTF32 + fused-tail path — then ReLU + Flatten can be folded into the heads'
        operand packs (linear.relu_flat_linear3x); else None.  (C, HW) is resolved lazily from the last conv.)"""
        if not (self.fused_relu_flatten and self.dense_3xtf32 and self.fused_dueling_tail and self.fuse_sibling_heads):
            return None
        name = self.first_conv_node()
        if name is None or not getattr(self, name).ends_with_relu_flatten() or name in self._outputs:
            return None
        users = [m for m in self._order if name in self._prev[m]]
        groups = {self._head_groups.get(u) for u in users}
        if len(groups) != 1 or None in groups:
            return None
        group = groups.pop()
        if sorted(users) != sorted(group) or group not in self._dueling:
            return None
        conv = list(getattr(self, name).children())[-3]
        adv, val = (getattr(self, self._dueling[group][r]) for r in ("adv", "val"))
        wa, wv = adv.MLP_2.weight, val.MLP_2.weight
        if wv.shape != (1, wa.shape[1]) or wa.shape[1] % 32 or wa.shape[1] > 1024 or wa.shape[0] > 32:
            return None                                   # the fused dueling tail (csrc/dueling.cu) would not take it
        k = adv.MLP_1.in_features
        c = conv.out_channels
        if k % c:
            return None
        return group, (c, k // c)

    def first_conv_node(self):
        """Name of the CNN2D node fed by external input 0, if it starts with the Atari conv_1."""
        for name in self._order:
            m = getattr(self, name)
            if isinstance(m, ConvStack) and self._ext[name] == [0] and not self._prev[name]:
                return name if m.is_atari_conv1() else None
        return None

    def first_stem_node(self):
        """Name of the RESCNN2D node fed by external input 0, if its stem is the one libb2rl's stem kernels run
        (the parallel of first_conv_node for the residual network)."""
        for name in self._order:
            m = getattr(self, name)
            if isinstance(m, ResidualStack) and self._ext[name] == [0] and not self._prev[name]:
                return name if m.is_fused_stem() else None
        return None

    def forward_from_stem(self, p, extra_inputs=()):
        """Forward pass given the stem's pooled output of the first RESCNN2D node (fused gather + stem kernel)."""
        name = self.first_stem_node()
        return self.forward([None, *extra_inputs], preset={name: getattr(self, name).forward_tail(p)})

    def forward_from_conv1(self, y, relu_applied: bool, extra_inputs=()):
        """Forward pass given conv_1's output of the first CNN2D node (fused gather+conv1 kernel)."""
        name = self.first_conv_node()
        stack = getattr(self, name)
        if y.is_cuda and self._prehead_group() is not None:
            from .linear import relu_flat_supported
            y_last = stack.forward_tail(y, relu_applied, stop_before_head=True)
            group = self._prehead_group()[0]
            ws = [getattr(self, n).MLP_1.weight for n in (self._dueling[group]["adv"], self._dueling[group]["val"])]
            if relu_flat_supported(y_last, ws):
                return self.forward([None, *extra_inputs], preset={name: _PreHead(y_last)})
            layers = list(stack.children())[-2:]                 # not channels_last after all: finish the stack
            feat = y_last
            for layer in layers:
                feat = stack._run(layer, feat)
            return self.forward([None, *extra_inputs], preset={name: feat})
        feat = stack.forward_tail(y, relu_applied)
        return self.forward([None, *extra_inputs], preset={name: feat})

    # -- the surface the learners call --------------------------------------------
    def getParameters(self):
        return list(self.parameters())

    def updateParameter(self, other: "GraphAgent", tau: float) -> None:
        with torch.no_grad():
            mine, theirs = list(self.parameters()), list(other.parameters())
            if tau == 1:
                torch._foreach_copy_(mine, theirs)
            else:
                torch._foreach_mul_(mine, 1 - tau)
                torch._foreach_add_(mine, theirs, alpha=tau)
        self.refresh_resident_heads()

    def calculateNorm(self):
        return sum(p.grad.norm(2) for p in self.parameters() if p.grad is not None)

    def clippingNorm(self, max_norm):
        torch.nn.utils.clip_grad_norm_(list(self.parameters()), max_norm)

    def _rec(self, name=None) -> Recurrent:
        return getattr(self, name or self._recurrent[0])

    def setCellState(self, hc, name=None):
        self._rec(name).set_state(hc)

    def getCellState(self, name=None):
        h, c = self._rec(name).state
        return h.clone(), c.clone()

    def detachCellState(self, name=None):
        self._rec(name).detach_state()

    def zeroCellState(self, num=1, name=None):
        self._rec(name).zero_state(num)
