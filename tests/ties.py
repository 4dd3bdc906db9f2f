"""Tie-dense single-layer graphs and an exact reference of their requantisation.

Every scale here is a power of two.  Then each step of the reference's float chain (acc * s_in * s_w, / s_out, the zero points,
the pooling divisor when the window area is a power of two) is exact in fp32, the value `t` the reference rounds is an exact
rational number, and exact ties (t = k + 1/2) occur by construction in a large share of the elements.  Ties are where the
kernels' fast epilogues (one multiply by M, round half to even with the MAGIC trick) differ from the reference's round() (half
away from zero), so they are where the tie guard and its rare path (common.cuh requant_fast*, gemm_tcgen05.cu fixq_*) must act.

`exact_layer` restates the reference's arithmetic in numpy: integer accumulators in int64, `t` in float64 (exact at these
scales), round half away from zero, then the clamp -- with each op's own placement of the zero point and rounding function, as
cited per op below (paths relative to the reference's source/device/cpu/op/; oracle/tb200_oracle.c restates the same lines).
It never calls the oracle library, so the CPU tests can pin the oracle against it.
"""
from dataclasses import dataclass, field

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

from tengine_b200 import abi
from tengine_b200.graphdef import GraphDef


def _pow2(s):
    m, _ = np.frexp(np.float64(s))
    return m == 0.5


def _round_away(t):
    return np.sign(t) * np.floor(np.abs(t) + 0.5)


@dataclass
class Rounding:
    """The last step of one layer: q = round(t) + add, then the clamp.  `t` already contains the zero point when the op adds it
    inside round() (`zp_inside`), in which case add == 0."""
    t: np.ndarray
    add: int
    lo: int
    hi: int
    zero: int = 0          # output zero point (uint8)
    zp_inside: bool = False
    below: str = "clamp"   # what happens below lo: "clamp", "wrap" (uint8 pool: no lower clamp, C cast), "to_hi" (int8 concat, sic)
    dtype: type = np.int8

    def bytes(self, rnd=_round_away, t=None, add=None):
        t = self.t if t is None else t
        q = rnd(t).astype(np.int64) + (self.add if add is None else add)
        q = np.where(q > self.hi, self.hi, q)
        if self.below == "clamp":
            q = np.where(q < self.lo, self.lo, q)
        elif self.below == "to_hi":
            q = np.where(q < self.lo, self.hi, q)
        return (q & 0xFF).astype(np.uint8).view(self.dtype) if self.dtype == np.int8 else (q & 0xFF).astype(np.uint8)

    def exact(self):
        return self.bytes()

    def half_even(self):
        """What a kernel without the tie guard computes: round half to even."""
        return self.bytes(np.rint)

    def zp_swapped(self):
        """The other placement of the output zero point (inside vs outside round()); differs from exact() only at negative ties."""
        if self.zp_inside:
            return self.bytes(t=self.t - self.zero, add=self.zero)
        return self.bytes(t=self.t + self.zero, add=0)

    def tie_mask(self):
        return np.abs(self.t - np.floor(self.t)) == 0.5

    def live_ties(self):
        """Exact ties whose rounding direction changes the output byte (ties that survive the clamp)."""
        lo = self.bytes(np.floor)
        hi = self.bytes(np.ceil)
        return self.tie_mask() & (lo != hi)


# ---- integer accumulators --------------------------------------------------------------------------------------------------
def conv_acc(x, w, L, zx=0, zw=0):
    """sum (x - zx)(w - zw) over the in-bounds taps (padding taps contribute 0: conv_kernel_ref_int8.c:104-121,
    conv_kernel_ref_uint8.c:167-181), exact: float64 GEMM of integers < 2^53."""
    xs = x.astype(np.float64) - zx
    ws = w.astype(np.float64) - zw
    n, c, h, wd = x.shape
    oc, cg, kh, kw = w.shape
    G = L["group"]
    sh, sw, dh, dw = L["stride_h"], L["stride_w"], L["dilation_h"], L["dilation_w"]
    xp = np.pad(xs, ((0, 0), (0, 0), (L["pad_h0"], L["pad_h1"]), (L["pad_w0"], L["pad_w1"])))
    ekh, ekw = dh * (kh - 1) + 1, dw * (kw - 1) + 1
    win = sliding_window_view(xp, (ekh, ekw), axis=(2, 3))[:, :, ::sh, ::sw, ::dh, ::dw]  # n c oh ow kh kw
    oh = (h + L["pad_h0"] + L["pad_h1"] - ekh) // sh + 1
    ow = (wd + L["pad_w0"] + L["pad_w1"] - ekw) // sw + 1
    win = win[:, :, :oh, :ow]
    og = oc // G
    out = np.empty((n, oc, oh, ow), np.float64)
    for gi in range(G):
        a = win[:, gi * cg:(gi + 1) * cg].transpose(0, 2, 3, 1, 4, 5).reshape(n * oh * ow, cg * kh * kw)
        b = ws[gi * og:(gi + 1) * og].reshape(og, cg * kh * kw)
        out[:, gi * og:(gi + 1) * og] = (a @ b.T).reshape(n, oh, ow, og).transpose(0, 3, 1, 2)
    return np.rint(out).astype(np.int64)


def _act_hcl(f, act):
    # conv/x86/conv_kernel_x86.c:1841-1889 (int8), :1745-1789 (uint8)
    if act == 0:
        f = np.maximum(f, 0)
    if act > 0:
        f = np.clip(f, 0, 6)
    return f


def _act_ref(f, act):
    # conv/conv_kernel_ref_int8.c:142-167, conv_kernel_ref_uint8.c:164-178
    if act >= 0:
        if act != 1:
            f = np.maximum(f, 0)
        if act == 1:
            f = np.clip(f, -1, 1)
        if act == 6:
            f = np.minimum(f, 6)
    return f


def _pool_windows(L, H, W, OH, OW):
    """pooling_kernel_ref_int8.c:84-120 window bounds and divisor per output pixel (as tb200_oracle.c pool_window)."""
    out = []
    for ph in range(OH):
        for pw in range(OW):
            hs = ph * L["stride_h"] - L["pad_h0"]
            he = min(hs + L["kernel_h"], H + L["pad_h0"])
            ws = pw * L["stride_w"] - L["pad_w0"]
            we = min(ws + L["kernel_w"], W + L["pad_w0"])
            psz = (he - hs) * (we - ws)
            hs, ws, he, we = max(hs, 0), max(ws, 0), min(he, H), min(we, W)
            if not L["caffe_flavor"]:
                psz = (he - hs) * (we - ws)
            out.append((ph, pw, hs, he, ws, we, psz))
    return out


def exact_layer(g, L, bufs):
    """Rounding step of layer L (a dict of g.layers) given the int8/uint8 arrays of its inputs in `bufs` (tensor id -> array)."""
    u8 = g.data_type == abi.DT_UINT8
    tin, tout = g.tensors[L["inputs"][0]], g.tensors[L["output"]]
    for t in [tout] + [g.tensors[i] for i in L["inputs"]]:
        assert _pow2(t["scale"]), "exact reference needs power-of-two scales"
    si, so = np.float64(tin["scale"]), np.float64(tout["scale"])
    zi, zo = tin["zero_point"], tout["zero_point"]
    x = bufs[L["inputs"][0]]
    i8 = dict(lo=-127, hi=127, dtype=np.int8)
    u8c = dict(lo=0, hi=255, dtype=np.uint8, zero=zo)
    op = L["op"]
    if op in (abi.OP_CONV, abi.OP_FC):
        ws = L["weight_scales"].astype(np.float64)
        assert all(_pow2(s) for s in ws)
        if op == abi.OP_FC:
            n = x.shape[0]
            xw = x.reshape(n, 1, 1, -1)
            w = L["weight"].reshape(L["weight"].shape[0], 1, 1, -1)
            acc = conv_acc(xw, w, dict(group=1, stride_h=1, stride_w=1, dilation_h=1, dilation_w=1, pad_h0=0, pad_h1=0, pad_w0=0,
                                       pad_w1=0), zi if u8 else 0, L["weight_zero"] if u8 else 0)
        else:
            acc = conv_acc(x, L["weight"], L, zi if u8 else 0, L["weight_zero"] if u8 else 0)
        oc = acc.shape[1]
        b = (L["bias"].astype(np.int64) if L["bias"] is not None else np.zeros(oc, np.int64)).reshape(1, oc, 1, 1)
        if not u8:
            sw = ws.reshape(1, oc, 1, 1)
            if op == abi.OP_FC:
                # fc/fc_ref.c:225 rq = s_in*s_w/s_out; :252 roundf((acc + bias) * rq); no activation
                return Rounding(t=(acc + b) * (si * sw / so), add=0, **i8)
            f = (acc + b) * si * sw  # conv_kernel_x86.c:1834 / conv_kernel_ref_int8.c:140
            f = _act_hcl(f, L["activation"]) if L["recipe"] == abi.RECIPE_HCL else _act_ref(f, L["activation"])
            return Rounding(t=f / so, add=0, **i8)  # round(f / s_out), clamp +-127
        S = si * np.float64(L["weight_scales"][0])
        if op == abi.OP_FC:
            # fc/fc_ref.c:146-166: data = bias*bias_scale + sum ; round(data / s_out) + zp (zp outside)
            f = acc * S + b * np.float64(L["bias_scale"])
            return Rounding(t=f / so, add=zo, **u8c)
        f = acc * S + b * S  # conv_kernel_x86.c:1723,1740 / conv_kernel_ref_uint8.c:94
        f = _act_hcl(f, L["activation"]) if L["recipe"] == abi.RECIPE_HCL else _act_ref(f, L["activation"])
        # conv_kernel_x86.c:1789 (int)(round(f / s_out) + zp); conv_kernel_ref_uint8.c:181 round(f / s_out) + zp: zp outside
        return Rounding(t=f / so, add=zo, **u8c)
    if op == abi.OP_RELU:
        f = (x.astype(np.float64) - (zi if u8 else 0)) * si
        f = np.where(f < 0, f * np.float64(np.float32(L["negative_slope"])), f)
        if u8:
            # relu/relu_kernel_ref_uint8.c:85: round(f / s_out + zp) -- zp INSIDE round
            return Rounding(t=f / so + zo, add=0, zp_inside=True, **u8c)
        return Rounding(t=f / so, add=0, **i8)  # relu_kernel_ref_int8.c:80
    if op == abi.OP_ELTWISE:
        t1 = g.tensors[L["inputs"][1]]
        y = bufs[L["inputs"][1]]
        f0 = (x.astype(np.float64) - (zi if u8 else 0)) * si
        f1 = (y.astype(np.float64) - (t1["zero_point"] if u8 else 0)) * np.float64(t1["scale"])
        f = f0 + f1 if L["elt_type"] == abi.ELT_SUM else f0 * f1
        # eltwise/eltwise_ref.c (uint8 :311-583: round(f / s_out) + zp; int8 :585-845: round(f / s_out))
        return Rounding(t=f / so, add=zo, **u8c) if u8 else Rounding(t=f / so, add=0, **i8)
    if op == abi.OP_CONCAT:
        ts = []
        for i in L["inputs"]:
            ti = g.tensors[i]
            q = bufs[i].astype(np.float64)
            if u8:
                # concat_kernel_ref_uint8.c:82 roundf((q - zp_in) * (s_in/s_out) + zp_out): zp INSIDE round
                ts.append((q - ti["zero_point"]) * (np.float64(ti["scale"]) / so) + zo)
            else:
                ts.append(q * (np.float64(ti["scale"]) / so))  # concat_kernel_ref_int8.c:70-80 roundf(q * (s_in/s_out))
        t = np.concatenate(ts, axis=1)
        return Rounding(t=t, add=0, zp_inside=True, **u8c) if u8 else Rounding(t=t, add=0, below="to_hi", **i8)
    if op == abi.OP_POOL:
        N, C, H, W = x.shape
        OH, OW = tout["dims"][2], tout["dims"][3]
        xf = x.astype(np.float64) - (zi if u8 else 0)
        t = np.empty((N, C, OH, OW), np.float64)
        for ph, pw, hs, he, ws_, we, psz in _pool_windows(L, H, W, OH, OW):
            win = xf[:, :, hs:he, ws_:we]
            if L["pool_method"] == abi.POOL_MAX:
                t[:, :, ph, pw] = win.max(axis=(2, 3)) * si / so  # int8: round(mx * s_in/s_out); uint8 :131 dequant, max
            else:
                assert _pow2(psz), "average pooling: the divisor must be a power of two for an exact reference"
                t[:, :, ph, pw] = win.sum(axis=(2, 3)) * si / psz / so
        if u8:
            # pooling_kernel_ref_uint8.c:190-197 round(v / s_out) + zp, upper clamp only
            return Rounding(t=t, add=zo, below="wrap", **u8c)
        return Rounding(t=t, add=0, **i8)
    raise ValueError(abi.OP_NAMES[op])


def exact_run(g, inputs):
    """Every layer of g in order.  Returns ({tensor id: bytes}, {tensor id: Rounding})."""
    bufs = dict(zip(g.inputs, inputs))
    rs = {}
    for L in g.layers:
        r = exact_layer(g, L, bufs)
        bufs[L["output"]] = r.exact()
        rs[L["output"]] = r
    return bufs, rs


# ---- what the planner decides (engine.cu): the epilogue MODE of a conv / FC layer ---------------------------------------------
def planned_mode(g, L):
    """0 fast, 1 fast with the bias fused (int8 conv), 2 exact -- the choice of engine.cu's prerun (fuse_bias, u8_tc_fast,
    fast_int_ok) for a layer on the tensor-core path."""
    u8 = g.data_type == abi.DT_UINT8
    tin, tout = g.tensors[L["inputs"][0]], g.tensors[L["output"]]
    oc = tout["dims"][1]
    w = L["weight"].reshape(oc, -1).astype(np.int64)
    bias = L["bias"].astype(np.float64) if L["bias"] is not None else np.zeros(oc)
    ws = L["weight_scales"].astype(np.float64)
    M = np.float64(tin["scale"]) * (ws[0] if u8 else ws) / np.float64(tout["scale"])
    sumabs = np.abs(w - L["weight_zero"]).sum(1) if u8 else np.abs(w).sum(1)
    bound = ((255.0 if u8 else 128.0) * sumabs + np.abs(bias)) * np.abs(M) + 256.0
    if not (bound < 32000.0).all():
        return 2
    if u8:
        S = np.float32(tin["scale"]) * np.float32(ws[0])
        if L["op"] == abi.OP_FC and L["bias"] is not None and L["bias_scale"] not in (0.0, S):
            return 2
        return 2 if (np.abs(bias * M) > 250.0).any() else 0
    if L["op"] == abi.OP_FC:
        return 0
    return 1 if (np.abs(bias * M) <= 100.0).all() else 0


# ---- builders --------------------------------------------------------------------------------------------------------------
# int8: s_in = 2^-4, s_out = 2^-6, s_w[c] = 2^-(m_c + 2) -> M_c = 2^-m_c.  The exponents are weighted towards 2^-1 / 2^-2 (where
# half / a quarter of all accumulators are ties) but cover every M from 2^-1 to 2^-8.
M_EXPS = (1, 1, 1, 2, 2, 3, 4, 5, 6, 7, 8)
S_IN, S_OUT = 2.0 ** -4, 2.0 ** -6
X_MAX = 15  # int8 inputs in [-15, 15]


@dataclass
class Case:
    name: str
    g: GraphDef
    inputs: list
    min_tie_frac: float = 0.10   # asserted lower bound of live ties / outputs of the last layer
    min_half_even_diff: int = 8  # asserted lower bound of bytes that round-half-to-even changes (last layer)
    mode: int = None             # planned epilogue MODE of the conv / FC layer (None: glue op)
    notes: dict = field(default_factory=dict)


def _amp(M, k, target=40.0, xstd=X_MAX / np.sqrt(3)):
    """Weight amplitude A (weights uniform in [-A, A]) that gives t = acc*M a spread of about `target`."""
    return int(np.clip(round(target / (M * np.sqrt(k) * xstd * 0.58)), 1, 127))


def _int8_weights(rng, oc, kshape, k, m_exps=M_EXPS):
    m = np.array([m_exps[c % len(m_exps)] for c in range(oc)])
    ws = (2.0 ** -(m + 2)).astype(np.float32)
    w = np.empty((oc,) + kshape, np.int8)
    for c in range(oc):
        a = _amp(2.0 ** -m[c], k)
        w[c] = rng.integers(-a, a + 1, kshape)
    return w, ws, m


def _int8_bias(rng, oc, m, mode):
    """Bias with |bias*M| <= 60 on every channel (fused: MODE 1), or one channel pushed past 100 (MODE 0), or None."""
    if mode is None:
        return None
    b = np.array([rng.integers(-60, 61) * 2 ** int(m[c]) + rng.integers(-2 ** int(m[c]) + 1, 2 ** int(m[c])) for c in range(oc)])
    b = np.clip(b, -60 * 2 ** m, 60 * 2 ** m)
    if mode == 0:
        c = 1 % oc
        b[c] = int(-101.5 * 2 ** int(m[c]))  # t of this channel shifted by -101.5: still mostly unclamped, the rest stays fused-size
    return b.astype(np.int32)


def int8_conv(rng, n, c, h, w, oc, k=1, stride=1, pad=0, group=1, activation=-1, recipe=abi.RECIPE_HCL, mode=1, name=None,
              x_max=X_MAX, m_exps=M_EXPS):
    """mode 1: fused bias; 0: one channel with |bias*M| > 100; 2: channel 0 is "hot" (weights +-127 at M = 2^-1: the
    clamp-range bound passes 32000 and the layer takes the exact epilogue; that channel saturates, the rest do not).
    m_exps: the exponents m of M_c = 2^-m dealt to the channels in turn."""
    g = GraphDef(abi.DT_INT8)
    x = g.input(n, c, h, w, S_IN)
    cg = c // group
    kk = cg * k * k
    wq, ws, m = _int8_weights(rng, oc, (cg, k, k), kk, m_exps)
    if mode == 2:
        m[0] = 1
        ws[0] = 2.0 ** -3
        wq[0] = rng.choice(np.array([-127, 127], np.int8), (cg, k, k))
    b = _int8_bias(rng, oc, m, 1 if mode == 2 else mode)
    y = g.conv(x, wq, b, ws, S_OUT, stride=stride, pad=pad, group=group, activation=activation, recipe=recipe)
    g.mark_output(y)
    xin = rng.integers(-x_max, x_max + 1, (n, c, h, w)).astype(np.int8)
    cs = Case(name or f"int8_conv_n{n}c{c}_{h}x{w}_oc{oc}_k{k}s{stride}p{pad}g{group}_a{activation}_r{recipe}_m{mode}", g, [xin])
    cs.mode = planned_mode(g, g.layers[0])
    assert cs.mode == mode, (cs.name, cs.mode)
    # ReLU layers lose the negative half of their ties to the clamp
    cs.min_tie_frac = 0.05 if activation >= 0 else 0.10
    return cs


def int8_fc(rng, n, k, oc, mode=0, name=None):
    """FC: roundf(acc * rq) with rq = M exactly (fc_ref.c:252); mode 2 through a hot channel as for int8_conv."""
    g = GraphDef(abi.DT_INT8)
    x = g.input(n, k, 1, 1, S_IN)
    wq, ws, m = _int8_weights(rng, oc, (k,), k)
    if mode == 2:
        m[0] = 1
        ws[0] = 2.0 ** -3
        wq[0] = rng.choice(np.array([-127, 127], np.int8), k)
    b = _int8_bias(rng, oc, m, 1)
    y = g.fc(x, wq, b, ws, S_OUT)
    g.mark_output(y)
    xin = rng.integers(-X_MAX, X_MAX + 1, (n, k, 1, 1)).astype(np.int8)
    cs = Case(name or f"int8_fc_n{n}_k{k}_oc{oc}_m{mode}", g, [xin])
    cs.mode = planned_mode(g, g.layers[0])
    assert cs.mode == mode, (cs.name, cs.mode)
    cs.min_half_even_diff = 4 if n * oc < 200 else 8
    return cs


# uint8: s_in = 2^-4, s_w = 2^-3, s_out = 2^-5 -> M = 2^-2 (a quarter of the accumulators are ties); zero points 128 / 100 / 110
U8_ZX, U8_ZW, U8_ZO = 128, 100, 110


def uint8_conv(rng, n, c, h, w, oc, k=1, stride=1, pad=0, group=1, activation=-1, recipe=abi.RECIPE_HCL, mode=0, fc=False,
               name=None, s_out=2.0 ** -5):
    """Zero points on input, weights and output; t spans about [-100, 100] around the output zero point, so negative ties are as
    common as positive ones.  mode 2: channel 0's bias has |bias*M| > 250 (that channel saturates)."""
    g = GraphDef(abi.DT_UINT8)
    s_in, s_w = 2.0 ** -4, 2.0 ** -3
    M = s_in * s_w / s_out
    x = g.input(n, c, h, w, s_in, U8_ZX)
    cg = c // group
    kk = (cg * k * k) if not fc else c * h * w
    a = max(1, min(100, int(round(35.0 / (M * np.sqrt(kk) * 6 * 0.58)))))
    while a > 1 and 255.0 * kk * a * (a + 1) / (2 * a + 1) * M > 28000:  # keep the clamp-range proof (planned_mode) passing
        a -= 1
    shape = (oc, kk) if fc else (oc, cg, k, k)
    wq = (U8_ZW + rng.integers(-a, a + 1, shape)).astype(np.uint8)
    b = (rng.integers(-40, 41, oc) / M + rng.integers(-3, 4, oc)).astype(np.int32)
    if mode == 2:
        b[0] = int(260 / M)
    if fc:
        y = g.fc(x, wq, b, [s_w], s_out, U8_ZO, weight_zero=U8_ZW)
    else:
        y = g.conv(x, wq, b, [s_w], s_out, U8_ZO, stride=stride, pad=pad, group=group, activation=activation, recipe=recipe,
                   weight_zero=U8_ZW)
    g.mark_output(y)
    xin = (U8_ZX + rng.integers(-10, 11, (n, c, h, w))).astype(np.uint8)
    kind = "fc" if fc else f"conv_k{k}s{stride}p{pad}g{group}_a{activation}_r{recipe}"
    cs = Case(name or f"uint8_{kind}_n{n}c{c}_{h}x{w}_oc{oc}_m{mode}", g, [xin])
    cs.mode = planned_mode(g, g.layers[0])
    assert cs.mode == mode, (cs.name, cs.mode)
    cs.min_tie_frac = 0.05 if activation >= 0 else 0.10
    return cs


# ---- glue ops -------------------------------------------------------------------------------------------------------------
def _in(rng, u8, shape, lo=-60, hi=60, zp=0):
    if u8:
        return (zp + rng.integers(lo, hi + 1, shape)).astype(np.uint8)
    return rng.integers(lo, hi + 1, shape).astype(np.int8)


def eltwise(rng, u8, elt, shape=(2, 24, 9, 11)):
    """SUM: t = a + b/2 (ties at odd b); PROD: t = a*b/16 (ties at a*b = 8 mod 16)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    z0, z1, zo = (120, 130, 110) if u8 else (0, 0, 0)
    s0, s1, so = (2.0 ** -4, 2.0 ** -5, 2.0 ** -4) if elt == abi.ELT_SUM else (2.0 ** -3, 2.0 ** -3, 2.0 ** -2)
    a = g.input(*shape, s0, z0)
    b = g.input(*shape, s1, z1)
    g.mark_output(g.eltwise(a, b, so, zo, elt_type=elt))
    r = (-60, 60) if elt == abi.ELT_SUM else (-40, 40)
    xs = [_in(rng, u8, shape, *r, zp=z0), _in(rng, u8, shape, *r, zp=z1)]
    name = ("uint8" if u8 else "int8") + "_eltwise_" + ("sum" if elt == abi.ELT_SUM else "prod")
    return Case(name, g, xs, min_tie_frac=0.10 if elt == abi.ELT_SUM else 0.05)


def relu(rng, u8, slope_exp=None, shape=(2, 40, 7, 9)):
    """s_out = 2 s_in: t = x/2 on the positive side (ties at odd x); leaky slope 2^-k: t = x/2^(k+1) below zero.
    uint8 adds the zero point inside round() (relu_kernel_ref_uint8.c:85)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi, zo = (128, 110) if u8 else (0, 0)
    x = g.input(*shape, 2.0 ** -5, zi)
    slope = 0.0 if slope_exp is None else 2.0 ** -slope_exp
    g.mark_output(g.relu(x, 2.0 ** -4, zo, negative_slope=slope))
    xs = [_in(rng, u8, shape, -100, 100, zp=zi)]
    name = ("uint8" if u8 else "int8") + ("_relu" if slope_exp is None else f"_leaky_relu_2^-{slope_exp}")
    return Case(name, g, xs, min_tie_frac=0.20)


def pool(rng, u8, method, kernel, stride, pad=0, caffe=0, global_pool=False, shape=(2, 20, 8, 10), scale_ratio=1):
    """Average pooling over power-of-two window areas (every divisor, also at padded borders, is 1, 2 or 4 for 2x2 windows; global
    pooling over 4x4 with s_out = s_in/4: t = sum/4); max pooling with s_out = 2 s_in (t = max/2)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi, zo = (128, 100) if u8 else (0, 0)
    x = g.input(*shape, 2.0 ** -4, zi)
    so = 2.0 ** -4 * scale_ratio
    y = g.pool(x, method, kernel, stride, pad, out_scale=so, out_zero=zo, global_pool=global_pool, caffe_flavor=caffe)
    g.mark_output(y)
    xs = [_in(rng, u8, shape, -90, 90, zp=zi)]
    name = (("uint8" if u8 else "int8") + ("_maxpool" if method == abi.POOL_MAX else "_avgpool") +
            (f"_global{shape[2]}x{shape[3]}" if global_pool else f"_k{kernel}s{stride}p{pad}_caffe{caffe}") + f"_r{scale_ratio}")
    return Case(name, g, xs, min_tie_frac=0.10)


def concat(rng, u8, shape=(2, 16, 6, 7), c2=32):
    """Two inputs with s_in / s_out = 1/2 and 1/4 (t = q/2, q/4)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    z0, z1, zo = (120, 135, 110) if u8 else (0, 0, 0)
    n, c, h, w = shape
    a = g.input(n, c, h, w, 2.0 ** -5, z0)
    b = g.input(n, c2, h, w, 2.0 ** -6, z1)
    g.mark_output(g.concat([a, b], 2.0 ** -4, zo))
    xs = [_in(rng, u8, (n, c, h, w), -100, 100, zp=z0), _in(rng, u8, (n, c2, h, w), -100, 100, zp=z1)]
    return Case(("uint8" if u8 else "int8") + f"_concat_c{c}_{c2}", g, xs, min_tie_frac=0.10)


def check_not_vacuous(case, rounding):
    """(a) enough live ties in the output; (b) round half to even changes enough bytes -- so a kernel without its tie guard
    fails this case."""
    frac = rounding.live_ties().mean()
    assert frac >= case.min_tie_frac, f"{case.name}: live ties {frac:.3f} < {case.min_tie_frac}"
    diff = int((rounding.exact() != rounding.half_even()).sum())
    assert diff >= case.min_half_even_diff, f"{case.name}: half-to-even changes only {diff} bytes"
    return frac, diff
