"""Seeded random graphs for the planner, and the planner's structural passes restated in Python.

`generate(seed, dtype)` builds a random DAG of 4-14 layers over every op GraphDef builds: each new layer draws its inputs from
every earlier tensor of a compatible shape, so values live long and fan out; a 3-channel graph input feeds a stem convolution
(which reads the NCHW input itself) and usually a layer that needs the NHWC copy too.  Node-fusion candidates are planted on
purpose, each as the pair that fuses and as pairs that miss exactly one clause of the fuse_nodes predicate.  Every output
scale is calibrated on the layer's own oracle result so that outputs are not saturated: a wrong byte cannot hide behind
clamping.

`plan(g, flags)` restates engine.cu sole_readers, fuse_nodes, the NHWC-copy and producer decisions of plan_kernels (with
plan_conv's stem predicate) and plan_activation_arena, line by line.  It only describes what the library decides, so that the
CPU test can show which planner edges the generated graphs reach (`COVERAGE`, with the `UNREACHABLE` ones and why) and the GPU
test can tie the restatement to the library through the plan lines TB200_DEBUG_LAUNCH prints.
"""
from dataclasses import dataclass, field

import numpy as np

from tengine_b200 import abi
from tengine_b200.graphdef import GraphDef, conv_out_dim
from tests.helpers import single_layer_graph

NOP = "nop"  # a layer folded into its producer or consumer (engine.cu TB200_OP_NOP_)
LUT2 = "lut2"  # sigmoid * x as one byte table (TB200_OP_LUT2_)


def cpad(c):
    return (c + 15) // 16 * 16  # common.cuh cpad


def align_up(v, a):
    return (v + a - 1) // a * a


# ---- what the restatement reports: one key per planner edge --------------------------------------------------------------------
COVERAGE = (
    [f"fuse_elt_relu:{k}" for k in ("fused", "second_reader", "is_output", "scale_differs", "zp_differs", "u8_c_mod16", "slope")]
    + [f"fuse_relu_pool:{k}" for k in ("fused", "second_reader", "is_output", "scale_differs", "zp_differs", "slope_negative", "slope_above_1",
                                        "not_max")]
    + [f"fuse_silu:{k}" for k in ("fused_operand0", "fused_operand1", "second_reader", "is_output", "not_prod", "post_relu", "other_operand")]
    + [f"arena:{k}" for k in ("reused_slot", "coalesced_left", "coalesced_right", "grew_trailing_block", "dead_value", "no_slot",
                              "reshape_scratch")]
    + ["inputs:nchw_only", "inputs:nchw_and_nhwc", "inputs:input_is_output", "outputs:read_later", "concat_same_tensor_twice",
       "eltwise_same_tensor"]
)

# keys a dtype cannot reach, and why
UNREACHABLE = {
    abi.DT_INT8: {
        "fuse_elt_relu:u8_c_mod16": "the C % 16 clause is for uint8 only: int8 pad lanes are 0, which ReLU keeps",
        "fuse_elt_relu:zp_differs": "int8 tensors are symmetric (zero point 0), so only the scale can differ",
        "fuse_relu_pool:zp_differs": "int8 tensors are symmetric (zero point 0), so only the scale can differ",
    },
    abi.DT_UINT8: {},
}


# ---- the restatement -------------------------------------------------------------------------------------------------------------
def sole_readers(layers, num_tensors, outputs):
    """engine.cu sole_readers: [tensor] the one layer that reads it, or -1 (no reader, several, or a graph output)."""
    count, reader = [0] * num_tensors, [-1] * num_tensors
    for li, L in enumerate(layers):
        for t in L["inputs"]:
            count[t] += 1
            reader[t] = li
    for t in range(num_tensors):
        if count[t] != 1:
            reader[t] = -1
    for t in outputs:
        reader[t] = -1
    return reader


def _readers(layers, t):
    return [li for li, L in enumerate(layers) if t in L["inputs"]]


def _quant_reason(ta, tb):
    if ta["scale"] != tb["scale"]:
        return "scale_differs"
    if ta["zero_point"] != tb["zero_point"]:
        return "zp_differs"
    return None


def fuse_nodes(g, fused, lp, pairs, keys):
    """engine.cu fuse_nodes: `fused` (copies of g.layers) is rewritten in place.  For every candidate pair it adds the key of the
    first clause that fails, or of the fusion."""
    T = g.tensors
    u8 = g.data_type == abi.DT_UINT8
    nt = len(T)
    # Eltwise -> ReLU
    orig = [dict(L, inputs=list(L["inputs"])) for L in fused]
    sole = sole_readers(orig, nt, g.outputs)
    for li, E in enumerate(orig):
        if E["op"] != abi.OP_ELTWISE or not any(orig[r]["op"] == abi.OP_RELU for r in _readers(orig, E["output"])):
            continue
        lj = sole[E["output"]]
        R = orig[lj] if lj > li else None
        if E["output"] in g.outputs:
            why = "is_output"
        elif R is None:
            why = "second_reader"
        elif R["op"] != abi.OP_RELU:
            continue
        elif R["negative_slope"] != 0.0:
            why = "slope"
        else:
            why = _quant_reason(T[E["output"]], T[R["output"]])
            if why is None and u8 and T[E["output"]]["dims"][1] % 16:
                why = "u8_c_mod16"
            if why is None and T[E["output"]]["dims"] != T[R["output"]]["dims"]:
                why = "dims"
        keys.add(f"fuse_elt_relu:{why or 'fused'}")
        if why:
            continue
        fused[li]["output"] = R["output"]
        lp[li]["post_relu"] = 1
        fused[lj]["op"], fused[lj]["inputs"] = NOP, []
        pairs.append(("elt_relu", li, lj))
    # (Leaky) ReLU -> max pooling
    sole = sole_readers(fused, nt, g.outputs)
    for li, R in enumerate(fused):
        if R["op"] != abi.OP_RELU or not any(fused[r]["op"] == abi.OP_POOL for r in _readers(fused, R["output"])):
            continue
        lj = sole[R["output"]]
        if R["output"] in g.outputs:
            why = "is_output"
        elif lj <= li:
            why = "second_reader"
        elif R["negative_slope"] < 0.0:
            why = "slope_negative"
        elif R["negative_slope"] > 1.0:
            why = "slope_above_1"
        elif fused[lj]["op"] != abi.OP_POOL:
            continue
        elif fused[lj]["pool_method"] != abi.POOL_MAX:
            why = "not_max"
        else:
            why = _quant_reason(T[R["output"]], T[fused[lj]["output"]])
        keys.add(f"fuse_relu_pool:{why or 'fused'}")
        if why:
            continue
        lp[lj]["pool_relu"] = li
        fused[lj]["inputs"][0] = R["inputs"][0]
        fused[li]["op"], fused[li]["inputs"] = NOP, []
        pairs.append(("relu_pool", lj, li))
    # Sigmoid -> Eltwise-PROD with the Sigmoid's own input
    sole = sole_readers(fused, nt, g.outputs)
    for li, S in enumerate(fused):
        if S["op"] != abi.OP_SIGMOID or not any(fused[r]["op"] == abi.OP_ELTWISE for r in _readers(fused, S["output"])):
            continue
        lj = sole[S["output"]]
        if S["output"] in g.outputs:
            why = "is_output"
        elif lj <= li:
            why = "second_reader"
        elif fused[lj]["op"] != abi.OP_ELTWISE:
            continue
        else:
            E = fused[lj]
            if E["elt_type"] != abi.ELT_PROD or len(E["inputs"]) != 2:
                why = "not_prod"
            elif lp[lj]["post_relu"]:
                why = "post_relu"
            else:
                a, b = E["inputs"]
                other = b if a == S["output"] else (a if b == S["output"] else -1)
                why = "other_operand" if other != S["inputs"][0] else None
        if why:
            keys.add(f"fuse_silu:{why}")
            continue
        operand = 0 if fused[lj]["inputs"][0] == S["output"] else 1
        keys.add(f"fuse_silu:fused_operand{operand}")
        lp[lj]["silu_sig"], lp[lj]["silu_operand"] = li, operand
        fused[lj]["op"], fused[lj]["inputs"] = LUT2, [S["inputs"][0]]
        fused[li]["op"], fused[li]["inputs"] = NOP, []
        pairs.append(("silu", lj, li))


@dataclass
class TensorPlan:
    off: int = 0
    slot: int = 0  # slot bytes: align_up(NHWC bytes, 1 KiB)
    nhwc_bytes: int = 0
    producer: int = -1
    last_use: int = -1
    has_slot: bool = True
    nhwc_needed: bool = False


@dataclass
class Plan:
    layers: list  # the layers after fusion (op NOP: folded)
    pairs: list  # (pass, layer that runs the pair, folded layer)
    tensors: list  # TensorPlan per tensor
    scratch: dict  # reshape layer -> (off, bytes)
    act_bytes: int
    unshared_bytes: int
    keys: set = field(default_factory=set)

    def folded(self):
        return {li for li, L in enumerate(self.layers) if L["op"] == NOP}


def reads_nchw(g, L):
    """engine.cu plan_conv: the stem kinds read the NCHW graph input themselves -- the gather stem (C <= 3, 3x3 or 7x7, a
    tensor-core kernel allowed) and the direct stem (C <= 4, group 1); both need group 1 and C <= 4, whatever the flags."""
    t = L["inputs"][0]
    return L["op"] == abi.OP_CONV and t in g.inputs and g.dims(t)[1] <= 4 and L["group"] == 1


def plan(g, flags=abi.PRERUN_DEFAULT):
    keys = set()
    nt = len(g.tensors)
    fused = [dict(L, inputs=list(L["inputs"])) for L in g.layers]
    lp = [dict(post_relu=0, pool_relu=-1, silu_sig=-1, silu_operand=0) for _ in fused]
    pairs = []
    if not flags & abi.PRERUN_NO_GRAPH:
        fuse_nodes(g, fused, lp, pairs, keys)
    # setup_tensors
    tp = []
    for t in g.tensors:
        n, c, h, w = t["dims"]
        nb = n * h * w * cpad(c)
        tp.append(TensorPlan(nhwc_bytes=nb, slot=align_up(nb, 1024)))
    # plan_kernels: producers, the NHWC copies of graph inputs, reshape kinds
    reshape = set()
    for li, L in enumerate(fused):
        if L["op"] == NOP:
            continue
        tp[L["output"]].producer = li
        stem = reads_nchw(g, L)
        for t in L["inputs"]:
            if t in g.inputs and not stem:
                tp[t].nhwc_needed = True
        if L["op"] == abi.OP_RESHAPE:
            (_, c, h, w), (_, oc, oh, ow) = g.dims(L["inputs"][0]), g.dims(L["output"])
            if not ((h * w == 1 and oh * ow == 1) or (c == oc and h == oh and w == ow)):
                reshape.add(li)
    for t in g.outputs:
        if t in g.inputs:
            tp[t].nhwc_needed = True
    # plan_activation_arena
    reuse = not flags & abi.PRERUN_NO_GRAPH
    for li, L in enumerate(fused):
        for t in L["inputs"]:
            tp[t].last_use = li
    free = []  # [off, bytes], sorted by offset
    top = 0

    def alloc(nbytes):
        nonlocal top
        for i, b in enumerate(free):
            if b[1] >= nbytes:
                off = b[0]
                b[0] += nbytes
                b[1] -= nbytes
                if not b[1]:
                    del free[i]
                keys.add("arena:reused_slot")
                return off
        if free and free[-1][0] + free[-1][1] == top:
            off = free.pop()[0]
            top = off + nbytes
            keys.add("arena:grew_trailing_block")
            return off
        off = top
        top += nbytes
        return off

    def release(off, nbytes):
        if not reuse or not nbytes:
            return
        i = 0
        while i < len(free) and free[i][0] < off:
            i += 1
        free.insert(i, [off, nbytes])
        if i + 1 < len(free) and free[i][0] + free[i][1] == free[i + 1][0]:
            free[i][1] += free[i + 1][1]
            del free[i + 1]
            keys.add("arena:coalesced_right")
        if i > 0 and free[i - 1][0] + free[i - 1][1] == free[i][0]:
            free[i - 1][1] += free[i][1]
            del free[i]
            keys.add("arena:coalesced_left")

    unshared = 0
    placed, freed = [False] * nt, [False] * nt
    for i, t in enumerate(tp):
        unshared += t.slot
        if t.producer < 0 and t.last_use < 0 and i not in g.inputs and i not in g.outputs:
            placed[i], t.has_slot = True, False
            unshared -= t.slot
            keys.add("arena:no_slot")
            continue
        if t.producer < 0:
            t.off, placed[i] = alloc(t.slot), True

    def permanent(i):
        return i in g.inputs or i in g.outputs or tp[i].producer < 0

    scratch = {}
    for li, L in enumerate(fused):
        if L["op"] == NOP:
            continue
        o = L["output"]
        if not placed[o]:
            tp[o].off, placed[o] = alloc(tp[o].slot), True
        if li in reshape:
            sb = align_up(int(np.prod(g.dims(o))), 1024)
            scratch[li] = (alloc(sb), sb)
            unshared += sb
            release(scratch[li][0], sb)
            keys.add("arena:reshape_scratch")
        for t in L["inputs"]:
            if tp[t].last_use == li and not permanent(t) and not freed[t]:
                release(tp[t].off, tp[t].slot)
                freed[t] = True
        if tp[o].last_use < li and not permanent(o) and not freed[o]:
            release(tp[o].off, tp[o].slot)
            freed[o] = True
            keys.add("arena:dead_value")
    # the structural keys
    for t in g.inputs:
        stem = any(L["op"] != NOP and reads_nchw(g, L) and L["inputs"][0] == t for L in fused)
        if stem:
            keys.add("inputs:nchw_and_nhwc" if tp[t].nhwc_needed else "inputs:nchw_only")
        if t in g.outputs:
            keys.add("inputs:input_is_output")
    for t in g.outputs:
        if tp[t].producer >= 0 and tp[t].last_use > tp[t].producer:
            keys.add("outputs:read_later")
    for L in g.layers:
        if L["op"] == abi.OP_CONCAT and len(set(L["inputs"])) < len(L["inputs"]):
            keys.add("concat_same_tensor_twice")
        if L["op"] == abi.OP_ELTWISE and L["inputs"][0] == L["inputs"][1]:
            keys.add("eltwise_same_tensor")
    return Plan(fused, pairs, tp, scratch, top, unshared, keys)


def live_ranges(g, p):
    """[first, last] layer index of every tensor with a slot, from the graph after fusion alone: producer to last reader (a value
    nobody reads lives at its producer only).  Graph inputs are live throughout, graph outputs from their producer to the end
    (their bytes are only read after the last layer).  Plus the reshape scratch, live in its layer.  Returns
    [(name, first, last, off, bytes)] with the bytes the tensor really occupies (NHWC)."""
    end = len(p.layers)
    out = []
    for i, t in enumerate(g.tensors):
        tpi = p.tensors[i]
        if not tpi.has_slot:
            continue
        prod = [li for li, L in enumerate(p.layers) if L["op"] != NOP and L["output"] == i]
        reads = [li for li, L in enumerate(p.layers) if i in L["inputs"]]
        if i in g.inputs or not prod:
            lo, hi = 0, end
        else:
            lo = prod[0]
            hi = end if i in g.outputs else max(reads + [lo])
        n, c, h, w = t["dims"]
        out.append((f"tensor {i}", lo, hi, tpi.off, n * h * w * cpad(c)))
    for li, (off, nb) in p.scratch.items():
        out.append((f"scratch of layer {li}", li, li, off, nb))
    return out


# ---- the generator -------------------------------------------------------------------------------------------------------------
@dataclass
class Meta:
    seed: int
    dtype: int
    planted: list = field(default_factory=list)  # (pattern, variant)


_OCS = (8, 12, 16, 20, 24, 32, 40, 48, 64, 96)
MAC_BUDGET = 3_000_000  # per convolution: keeps the CPU oracle at milliseconds per graph


class _Gen:
    def __init__(self, seed, dtype, batch=None):
        from oracle.pyoracle import Oracle

        self.rng = np.random.default_rng([seed, dtype])
        self.u8 = dtype == abi.DT_UINT8
        self.g = GraphDef(dtype)
        self.n = int(self.rng.integers(1, 6))
        if batch:
            self.n = batch
        self.data_rng = np.random.default_rng([seed, dtype, self.n, 1])
        self.vals = {}
        self.hidden = set()  # the middle tensors of planted pairs: no other layer reads them, none becomes an output by chance
        self.oracle = Oracle()
        self.meta = Meta(seed, dtype)
        self.max_layers = int(self.rng.integers(4, 15))

    # -- helpers --
    def choice(self, seq):
        return seq[int(self.rng.integers(0, len(seq)))]

    def coin(self, p):
        return self.rng.random() < p

    def zp(self, signed=True):
        if not self.u8:
            return 0
        return int(self.rng.integers(110, 146)) if signed else int(self.rng.integers(16, 48))

    def unit_range(self):
        """(scale, zero point) of a sigmoid or softmax output: [0, 1] inside the range, clear of its ends."""
        return (1 / 225, 15) if self.u8 else (1 / 120, 0)

    def rms_real(self, t):
        T = self.g.tensors[t]
        v = self.vals[t].astype(np.float64) - T["zero_point"]
        return max(float(np.sqrt((v * v).mean())) * T["scale"], 1e-4)

    def tensors(self, pred=lambda d: True):
        return [t for t in range(len(self.g.tensors)) if t in self.vals and t not in self.hidden and pred(self.g.dims(t))]

    def room(self, k):
        return len(self.g.layers) + k <= self.max_layers

    def add_input(self, c, h, w, scale):
        t = self.g.input(self.n, c, h, w, scale, self.zp())
        d = (self.n, c, h, w)
        self.vals[t] = (self.data_rng.integers(0, 256, d).astype(np.uint8) if self.u8 else
                        self.data_rng.integers(-127, 128, d).astype(np.int8))
        return t

    def _run_last(self):
        h, ids = single_layer_graph(self.g, len(self.g.layers) - 1)
        return self.oracle.run(h, [self.vals[t] for t in ids], uint8_mode=0)[h.outputs[0]]

    def saturated(self, q):
        return float(((q == 0) | (q == 255)).mean()) if self.u8 else float((np.abs(q.astype(np.int32)) >= 127).mean())

    def emit(self, build, scale, zp, calibrate=True):
        """build(scale, zero point) appends one layer; its output scale is widened while more than 4 % of the bytes saturate, and
        narrowed while the bytes spread over too few values."""
        for _ in range(5):
            t = build(float(scale), int(zp))
            q = self._run_last()
            if not calibrate:
                break
            spread = float(q.astype(np.float64).std())
            if self.saturated(q) > 0.04:
                scale *= 2.5
            elif spread < 6 and q.size > 16:
                scale /= 2.5
            else:
                break
            self.g.layers.pop()
            self.g.tensors.pop()
        self.vals[t] = q
        return t

    # -- ops --
    def conv(self, x, oc=None, k=None, s=None, kind=None, activation=None):
        g, rng = self.g, self.rng
        n, c, h, w = g.dims(x)
        if kind is None:
            kinds = ["dense"] * 4
            if c > 1 and x not in g.inputs:
                kinds += ["depthwise"]
            if c % 8 == 0:
                kinds += ["grouped"]
            kind = self.choice(kinds)
        group = c if kind == "depthwise" else (self.choice([2] + ([4] if c % 16 == 0 else [])) if kind == "grouped" else 1)
        if k is None:
            k = 3 if kind == "depthwise" else self.choice([1, 1, 3, 3, 5] if x not in g.inputs else [3, 3, 7, 1])
        if s is None:
            s = self.choice([1, 1, 2])
        p = k // 2
        if oc is None:
            oc = c if kind == "depthwise" else self.choice([o for o in _OCS if o % (4 * group) == 0] or [4 * group])
        oh, ow = conv_out_dim(h, k, s, p, p, 1), conv_out_dim(w, k, s, p, p, 1)
        while kind != "depthwise" and oc > 8 and n * oh * ow * oc * (c // group) * k * k > MAC_BUDGET and (oc // 2) % (4 * group) == 0:
            oc //= 2
        if kind != "depthwise" and n * oh * ow * oc * (c // group) * k * k > MAC_BUDGET:
            k, p = 1, 0
        cg = c // group
        if self.u8:
            wq, wz = rng.integers(0, 256, (oc, cg, k, k)).astype(np.uint8), int(rng.integers(112, 144))
            ws = np.array([0.004], np.float32)
            w_rms = 0.004 * float(np.sqrt(((wq.astype(np.float64) - wz) ** 2).mean()))
        else:
            wq, wz = rng.integers(-127, 128, (oc, cg, k, k)).astype(np.int8), 0
            ws = rng.uniform(0.001, 0.01, oc).astype(np.float32)
            w_rms = float(ws.mean()) * float(np.sqrt((wq.astype(np.float64) ** 2).mean()))
        if activation is None:
            activation = self.choice([-1, 0])
        std = max(np.sqrt(cg * k * k) * self.rms_real(x) * w_rms, 1e-4)
        sin = g.tensors[x]["scale"]
        bias = np.clip(rng.uniform(-0.5, 0.5, oc) * std / (sin * float(ws.mean())), -2 ** 20, 2 ** 20).astype(np.int32)
        depthwise = group == c and group == oc and group > 1
        recipe = abi.RECIPE_HCL if group == 1 else abi.RECIPE_REF
        if depthwise and not self.u8 and n == 1 and k == 3 and s in (1, 2):
            recipe = abi.RECIPE_HCL  # b200_device.cc conv_recipe: what the reference CPU device selects
        zp = self.zp(signed=activation != 0)
        return self.emit(lambda sc, z: g.conv(x, wq, bias, ws, sc, z, stride=s, pad=p, group=group, activation=activation,
                                              recipe=recipe, weight_zero=wz), std / 30, zp)

    def fc(self, x):
        g, rng = self.g, self.rng
        n, c, h, w = g.dims(x)
        oc = self.choice([10, 16, 24, 40])
        kk = c * h * w
        if self.u8:
            wq, wz, ws = rng.integers(0, 256, (oc, kk)).astype(np.uint8), int(rng.integers(112, 144)), np.array([0.004], np.float32)
            w_rms = 0.004 * float(np.sqrt(((wq.astype(np.float64) - wz) ** 2).mean()))
        else:
            wq, wz, ws = rng.integers(-127, 128, (oc, kk)).astype(np.int8), 0, rng.uniform(0.001, 0.01, oc).astype(np.float32)
            w_rms = float(ws.mean()) * float(np.sqrt((wq.astype(np.float64) ** 2).mean()))
        std = max(np.sqrt(kk) * self.rms_real(x) * w_rms, 1e-4)
        bias = np.clip(rng.uniform(-0.5, 0.5, oc) * std / (g.tensors[x]["scale"] * float(ws.mean())), -2 ** 20, 2 ** 20).astype(np.int32)
        return self.emit(lambda sc, z: g.fc(x, wq, bias, ws, sc, z, weight_zero=wz), std / 30, self.zp())

    def pool(self, x, method=None, out_scale=None, global_pool=None):
        g = self.g
        _, _, h, w = g.dims(x)
        method = self.choice([abi.POOL_MAX, abi.POOL_AVG]) if method is None else method
        opts = [(2, 2, 0), (3, 2, 1), (3, 1, 1)] if min(h, w) >= 3 else [(2, 2, 0)] if min(h, w) >= 2 else []
        if global_pool is None:
            global_pool = not opts or self.coin(0.15)
        k, s, p = (1, 1, 0) if global_pool else self.choice(opts)
        src = g.tensors[x]
        sc = src["scale"] if out_scale is None else out_scale
        return self.emit(lambda _s, _z: g.pool(x, method, k, s, p, out_scale=sc, out_zero=src["zero_point"], global_pool=global_pool),
                         sc, src["zero_point"], calibrate=False)

    def relu(self, x, slope=None, out_scale=None, out_zero=None):
        src = self.g.tensors[x]
        slope = self.choice([0.0, 0.0, 0.1]) if slope is None else slope
        sc = src["scale"] if out_scale is None else out_scale
        z = src["zero_point"] if out_zero is None else out_zero
        return self.emit(lambda _s, _z: self.g.relu(x, sc, z, negative_slope=slope), sc, z, calibrate=False)

    def eltwise(self, a, b, elt_type=None):
        g = self.g
        elt_type = self.choice([abi.ELT_SUM, abi.ELT_SUM, abi.ELT_PROD]) if elt_type is None else elt_type
        ra, rb = self.rms_real(a), self.rms_real(b)
        std = ra * rb if elt_type == abi.ELT_PROD else float(np.hypot(ra, rb))
        return self.emit(lambda sc, z: g.eltwise(a, b, sc, z, elt_type=elt_type), std / 30, self.zp())

    def same_dims(self, a):
        return self.tensors(lambda d: d == self.g.dims(a))

    # -- the random layer --
    def random_layer(self):
        g = self.g
        ops = ["conv"] * 5 + ["pool", "relu", "eltwise", "eltwise", "concat", "concat", "fc", "upsample", "identity", "softmax",
                                "sigmoid", "flatten"] + (["hardswish"] if self.u8 else [])
        op = self.choice(ops)
        spatial = self.tensors(lambda d: d[2] * d[3] > 1 and d[1] <= 160)
        if op == "conv":
            xs = self.tensors(lambda d: d[1] <= 160)
            return self.conv(self.choice(xs))
        if op == "fc":
            xs = self.tensors(lambda d: d[1] * d[2] * d[3] <= 1536)
            return self.fc(self.choice(xs)) if xs else None
        if op == "pool":
            return self.pool(self.choice(spatial)) if spatial else None
        x = self.choice(self.tensors())
        src = g.tensors[x]
        if op == "relu":
            if self.coin(0.4):
                return self.relu(x, out_scale=src["scale"] * 1.25, out_zero=src["zero_point"])
            return self.relu(x)
        if op == "eltwise":
            b = x if self.coin(0.25) else self.choice(self.same_dims(x))
            return self.eltwise(x, b)
        if op == "concat":
            n, _, h, w = g.dims(x)
            xs = [x]
            pool = self.tensors(lambda d: d[0] == n and d[2] == h and d[3] == w)
            for _ in range(int(self.rng.integers(0, 4))):
                cand = self.choice(pool)
                if sum(g.dims(t)[1] for t in xs) + g.dims(cand)[1] <= 192:
                    xs.append(cand)
            sc = max(g.tensors[t]["scale"] for t in xs) * self.choice([1.0, 1.3])
            zs = [g.tensors[t]["zero_point"] for t in xs]
            return self.emit(lambda s_, z_: g.concat(xs, s_, z_), sc, zs[0], calibrate=len(set(zs)) > 1 or sc != g.tensors[x]["scale"])
        if op == "upsample":
            xs = self.tensors(lambda d: d[2] <= 16 and d[3] <= 16 and d[1] <= 96)
            if not xs:
                return None
            y = self.choice(xs)
            return self.emit(lambda s_, z_: g.upsample(y, 2), 0, 0, calibrate=False)
        if op == "identity":
            return self.emit(lambda s_, z_: g.identity(x), 0, 0, calibrate=False)
        if op == "softmax":
            xs = self.tensors(lambda d: d[1] <= 128)
            y = self.choice(xs)
            return self.emit(lambda s_, z_: g.softmax(y, s_, z_), *self.unit_range(), calibrate=False)
        if op == "sigmoid":
            return self.emit(lambda s_, z_: g.sigmoid(x, s_, z_), *self.unit_range(), calibrate=False)
        if op == "hardswish":
            r = self.rms_real(x)
            return self.emit(lambda s_, z_: g.hardswish(x, s_, z_), 4 * r / 200, 50)
        if op == "flatten":
            xs = self.tensors(lambda d: d[1] * d[2] * d[3] <= 2048)
            y = self.choice(xs)
            return self.emit(lambda s_, z_: g.flatten(y), 0, 0, calibrate=False)
        raise AssertionError(op)

    def c16_tensor(self, mod16):
        """A tensor with C % 16 == 0 (mod16) or != 0: an existing one, else a new 1x1 convolution."""
        xs = self.tensors(lambda d: (d[1] % 16 == 0) == mod16 and d[2] * d[3] > 1)
        if xs and self.coin(0.6):
            return self.choice(xs)
        src = self.choice(self.tensors(lambda d: d[2] * d[3] > 1 and d[1] <= 160))
        return self.conv(src, oc=self.choice([16, 32, 48] if mod16 else [8, 20, 24, 40]), k=1, s=1, kind="dense")

    # -- planted fusion candidates: the pair that fuses and pairs that miss one clause --
    def plant_elt_relu(self):
        v = self.choice(["fused", "fused", "second_reader", "is_output", "scale_differs", "slope"] + (["zp_differs", "u8_c_mod16"] if self.u8 else []))
        a = self.c16_tensor(mod16=v != "u8_c_mod16" or not self.u8)
        b = self.choice(self.same_dims(a))
        e = self.eltwise(a, b, elt_type=abi.ELT_SUM if self.coin(0.7) else abi.ELT_PROD)
        self.hidden.add(e)
        src = self.g.tensors[e]
        sc, z = src["scale"], src["zero_point"]
        if v == "scale_differs":
            sc *= 1.25
        if v == "zp_differs":
            z += 3
        self.relu(e, slope=0.1 if v == "slope" else 0.0, out_scale=sc, out_zero=z)
        if v == "second_reader":
            self.pool(e, method=abi.POOL_AVG)
        if v == "is_output":
            self.g.mark_output(e)
        self.meta.planted.append(("elt_relu", v))

    def plant_relu_pool(self):
        v = self.choice(["fused", "fused", "second_reader", "is_output", "scale_differs", "slope_negative", "slope_above_1", "not_max"]
                        + (["zp_differs"] if self.u8 else []))
        xs = self.tensors(lambda d: d[2] >= 2 and d[3] >= 2 and d[1] <= 160)
        x = self.choice(xs)
        slope = {"slope_negative": -0.1, "slope_above_1": 1.5}.get(v, self.choice([0.0, 0.1, 1.0]))
        src = self.g.tensors[x]
        r = self.relu(x, slope=slope, out_scale=src["scale"] * self.choice([1.0, 1.5]), out_zero=src["zero_point"])
        self.hidden.add(r)
        rs = self.g.tensors[r]
        if v == "zp_differs":
            self.emit(lambda _s, _z: self.g.pool(r, abi.POOL_MAX, 2, 2, 0, out_scale=rs["scale"], out_zero=rs["zero_point"] + 4), 0, 0,
                      calibrate=False)
        else:
            self.pool(r, method=abi.POOL_AVG if v == "not_max" else abi.POOL_MAX, out_scale=rs["scale"] * (1.2 if v == "scale_differs" else 1.0),
                      global_pool=False if min(self.g.dims(r)[2:]) >= 2 else None)
        if v == "second_reader":
            self.emit(lambda _s, _z: self.g.identity(r), 0, 0, calibrate=False)
        if v == "is_output":
            self.g.mark_output(r)
        self.meta.planted.append(("relu_pool", v))

    def plant_silu(self):
        v = self.choice(["fused0", "fused1", "second_reader", "is_output", "other_operand", "not_prod", "post_relu"])
        x = self.c16_tensor(mod16=True) if self.u8 and v == "post_relu" else self.choice(self.tensors())
        s = self.emit(lambda s_, z_: self.g.sigmoid(x, s_, z_), *self.unit_range(), calibrate=False)
        self.hidden.add(s)
        other = x
        if v == "other_operand":
            other = self.emit(lambda _s, _z: self.g.identity(x), 0, 0, calibrate=False)
        a, b = (x, s) if v == "fused1" else (s, other)
        e = self.eltwise(a, b, elt_type=abi.ELT_SUM if v == "not_prod" else abi.ELT_PROD)
        if v == "post_relu":
            self.hidden.add(e)
            es = self.g.tensors[e]
            self.relu(e, slope=0.0, out_scale=es["scale"], out_zero=es["zero_point"])
        if v == "second_reader":
            self.relu(s)
        if v == "is_output":
            self.g.mark_output(s)
        self.meta.planted.append(("silu", v))

    def build(self):
        g = self.g
        h, w = int(self.rng.integers(6, 25)), int(self.rng.integers(6, 25))
        x0 = self.add_input(3, h, w, 0.02)
        extra = int(self.rng.integers(0, 3))
        for _ in range(extra):
            half = self.coin(0.4)
            self.add_input(self.choice([8, 16, 24, 32, 40]), (h + 1) // 2 if half else h, (w + 1) // 2 if half else w, 0.03)
        # the 3-channel input: a stem reads it as NCHW; usually a layer that needs its NHWC copy reads it too
        self.conv(x0, k=self.choice([3, 3, 7, 1]), kind="dense")
        if self.coin(0.7):
            self.choice([lambda: self.pool(x0), lambda: self.relu(x0), lambda: self.eltwise(x0, x0),
                         lambda: self.emit(lambda s_, z_: g.concat([x0, x0], s_, z_), 0.02, g.tensors[x0]["zero_point"], calibrate=False)])()
        if self.coin(0.15):
            g.mark_output(x0)
        plants = [self.plant_elt_relu, self.plant_relu_pool, self.plant_silu]
        while len(g.layers) < self.max_layers:
            if self.room(4) and self.coin(0.4):
                self.choice(plants)()
            else:
                self.random_layer()
        # outputs: the last tensor, sometimes a mid-graph tensor that later layers still read, sometimes an unread one
        last = g.layers[-1]["output"]
        if last not in g.outputs:
            g.mark_output(last)
        read = {t for L in g.layers for t in L["inputs"]}
        mids = [L["output"] for L in g.layers[:-1] if L["output"] in read and L["output"] not in set(g.outputs) | self.hidden]
        if mids and len(g.outputs) < 3 and self.coin(0.6):
            g.mark_output(self.choice(mids))
        unread = [L["output"] for L in g.layers if L["output"] not in read and L["output"] not in set(g.outputs) | self.hidden]
        if unread and len(g.outputs) < 3 and self.coin(0.3):
            g.mark_output(self.choice(unread))
        inputs = [self.vals[t] for t in g.inputs]
        return g, inputs, self.meta


def generate(seed, dtype, batch=None):
    """(GraphDef, inputs, Meta) of graph `seed`; `batch` rebuilds the same structure at another batch."""
    return _Gen(seed, dtype, batch).build()


def saturated_fraction(g, tensors):
    """Share of the bytes of the graph's outputs at the ends of the range."""
    tot = sat = 0
    for t in g.outputs:
        q = tensors[t]
        tot += q.size
        sat += int(((q == 0) | (q == 255)).sum()) if g.data_type == abi.DT_UINT8 else int((np.abs(q.astype(np.int32)) >= 127).sum())
    return sat / tot
