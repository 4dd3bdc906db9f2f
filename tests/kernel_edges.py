"""Single-layer cases at the edges of each kernel's tiling and of the planner's kernel choice, with the host-side plan geometry
restated in Python.

The tie-dense builders of tests/ties.py make the layers (power-of-two scales: `ties.exact_run` is an exact reference, independent
of the oracle); ops that `ties.exact_layer` does not cover (softmax, upsample, sigmoid) are compared with the oracle instead.

`gemm_geometry`, `dw_geometry` and `conv_kind` restate the C planners line by line (cited at each function).  They only describe
what the library decides -- no plan logic lives here -- so that the CPU test can show every entry reaches the geometry it is
meant to, and the GPU test can tie the restatement to the library (TB200_DEBUG_LAUNCH prints the GEMM's plan).

Every boundary is probed from both sides: an entry per side, listed in `BOUNDARIES`.
"""
from dataclasses import dataclass, field

import numpy as np

from tengine_b200 import abi
from tengine_b200.graphdef import GraphDef
from tests import ties


def cpad(c):
    return (c + 15) // 16 * 16  # common.cuh cpad


# ---- gemm_tcgen05.cu: plan geometry of the persistent GEMM ------------------------------------------------------------------
BLOCK_M, ACC_COLS_MAX, PAR_MAX, MAX_STAGES, B_RESIDENT_MAX = 128, 128, 2048, 24, 96 * 1024
EPI_WARPS, SMEM_CTL = 16, 432  # sizeof(GemmSmemCtl): (2 * MAX_STAGES + 5) uint64, 16-byte aligned


def _block_n(ocp):
    nt = (ocp + 127) // 128  # gemm_block_n
    return ((ocp + nt - 1) // nt + 15) & ~15


def gemm_geometry(ocp, u8zp, m=None, k=None, conv=None):
    """The plan of gemm_plan_create (flat: m rows, k = K) or gemm_plan_create_conv (conv = dict(n, h, w, cp, oh, ow, kh, kw,
    stride, ph0, pw0)).  u8zp is the planners' `u8` argument: 0 for int8, 1 + weight zero point for uint8.  Restates
    gemm_tcgen05.cu gemm_block_n (:823-829), gemm_plan_create (:884-908), gemm_plan_create_conv (:912-979), plan_stage
    (:835-843), epilogue_smem_bytes / plan_ring (:861-882), and launch_gemm_i8's par_all and BORDER (:1023, :1051)."""
    G = dict(ocp=ocp)
    bn = G["block_n"] = _block_n(ocp)
    G["n_tiles"] = n_tiles = (ocp + bn - 1) // bn
    G["n_uneven"] = ocp % bn != 0
    if conv is None:
        G["block_k"] = bk = 32 if k <= 32 else (64 if k <= 64 else 128)
        G["k_blocks"] = kb = (k + bk - 1) // bk
        G["cblocks"] = kb
        G["m_tiles"] = m_tiles = (m + BLOCK_M - 1) // BLOCK_M
        G["rows_valid"], G["out_mode"], G["m_rem"] = BLOCK_M, 0, m % BLOCK_M
        G["bw"] = G["bh"] = G["bn"] = None
        G["border"] = 0
    else:
        c = conv
        taps = c["kh"] * c["kw"]
        cp = c["cp"]
        if taps == 1:
            bk = 32 if cp <= 32 else (64 if cp <= 64 else 128)
        else:
            bk = 128 if cp % 128 == 0 else (64 if cp % 64 == 0 else 32)
        G["block_k"] = bk
        G["cblocks"] = cb = (cp + bk - 1) // bk
        G["k_blocks"] = kb = taps * cb
        G["taps"] = taps
        oh, ow, n = c["oh"], c["ow"], c["n"]
        if ow <= BLOCK_M:
            bw = ow
            bh = BLOCK_M // ow if BLOCK_M // ow < oh else oh
            bnn = BLOCK_M // (ow * oh) if bh == oh else 1
            bnn = max(1, min(bnn, n))
        else:
            bw, bh, bnn = BLOCK_M, 1, 1
        G["bw"], G["bh"], G["bn"] = bw, bh, bnn
        m_tiles = ((ow + bw - 1) // bw) * ((oh + bh - 1) // bh) * ((n + bnn - 1) // bnn)
        G["m_tiles"] = m_tiles
        G["rows_valid"] = bw * bh * bnn
        G["out_mode"] = 2 if bw != ow else (0 if bnn > 1 else 1)
        G["n_partial"] = bnn > 1 and n % bnn != 0
        G["oh_partial"] = oh % bh != 0
        s = c["stride"]
        pad_1x1 = c["ph0"] or c["pw0"] or (oh - 1) * s >= c["h"] or (ow - 1) * s >= c["w"]
        G["border"] = int(bool(u8zp) and (taps > 1 or bool(pad_1x1)))
        G["m_rem"] = None
    G["tail"] = G["rows_valid"] % 32
    mt = 1
    if n_tiles == 1:
        while mt < 4 and mt * 2 * bn <= ACC_COLS_MAX and mt * 2 <= m_tiles:
            mt *= 2
    G["mt"] = mt
    nch = bn // 16
    G["cs"] = cs = 2 if nch % 2 == 0 and (mt * (nch // 2)) % 4 == 0 else 1
    par_ch = n_tiles * bn
    G["par_all"] = 1 if par_ch <= PAR_MAX else 0
    cplane = u8zp > 1
    epi = EPI_WARPS * 2 * 512 * cs + (par_ch if par_ch <= PAR_MAX else bn) * 8 + SMEM_CTL + 2048 + 128 * (mt * bn * 4 + 16) + 16
    budget = 224 * 1024 - epi - (4096 if cplane else 0)
    a_bytes, b_al = BLOCK_M * bk, (bn * bk + 1023) & ~1023
    b_res = 1 if kb * b_al <= B_RESIDENT_MAX else 0
    if b_res and (budget - kb * b_al) // a_bytes < 3:
        b_res = 0
    G["b_res"] = b_res
    return G


# ---- dw_tma.cu dw_plan_create (:250-271): the TMA depthwise 3x3 or the generic kernel --------------------------------------
DW_CH = 32


def dw_geometry(u8, kh, kw, stride, oh, ow, dil=1):
    D = dict(valid=False, stride=stride, tw=None, gpr=None, rows_per_cta=None)
    if u8 or kh != 3 or kw != 3 or dil != 1 or stride not in (1, 2):
        return D
    D["tw"] = tw = 8 if stride == 1 else 4
    D["gpr"] = gpr = (ow + tw - 1) // tw
    if gpr > 16:
        return D
    rpc = 16 // gpr
    D["rows_capped"] = rpc > oh
    D["rows_per_cta"] = rpc = min(rpc, oh)
    tile_cols, tile_rows = (gpr * tw - 1) * stride + 3, (rpc - 1) * stride + 3
    if tile_cols > 256 or tile_rows > 256 or tile_rows * tile_cols * DW_CH > 48 * 1024:
        return D
    D["valid"] = True
    return D


# ---- engine.cu plan_conv (:768-809): the kernel of a convolution -----------------------------------------------------------
def conv_kind(g, L, no_tc=False):
    """'gemm', 'igemm', 'dw', 'direct', 'stem', 'gather' (NCHW stem / 16-channel input) or 'window32' (32-channel 3x3: decided by
    window_nhwc_fits, which is not restated: no entry here takes that branch)."""
    tin, tout = g.tensors[L["inputs"][0]], g.tensors[L["output"]]
    _, C, _, _ = tin["dims"]
    OC, OW = tout["dims"][1], tout["dims"][3]
    cp, ocp = cpad(C), cpad(OC)
    kh, kw, sh, sw, grp = L["kernel_h"], L["kernel_w"], L["stride_h"], L["stride_w"], L["group"]
    is_input = L["inputs"][0] in g.inputs
    tc = not no_tc and grp == 1
    plain = L["dilation_h"] == 1 and L["dilation_w"] == 1 and sh == sw
    k3 = kh == 3 and kw == 3
    gather = tc and plain and ocp <= 256
    nopad = not (L["pad_h0"] or L["pad_h1"] or L["pad_w0"] or L["pad_w1"])
    if is_input and C <= 3 and gather and kh == kw and kh in (3, 7):
        return "gather"
    if is_input and C <= 4 and grp == 1:
        return "stem"
    if gather and k3 and cp == 16:
        return "gather"
    if gather and k3 and cp == 32 and sh in (1, 2):
        return "window32"
    if grp == C and OC == C and C > 1:
        return "dw"
    if tc and kh == 1 and kw == 1 and sh == 1 and sw == 1 and nopad:
        return "gemm"
    if tc and plain and sh in (1, 2) and (kh * kw == 1 or cp % 32 == 0) and OW <= 4096 and kh * kw <= 64:
        return "igemm"
    return "direct"


def layer_geometry(g, L):
    """The restated plan of a conv / FC layer: dict with 'kind' and the kind's geometry."""
    u8 = g.data_type == abi.DT_UINT8
    n, C, Hh, W = g.tensors[L["inputs"][0]]["dims"]
    _, OC, OH, OW = g.tensors[L["output"]]["dims"]
    cp, ocp = cpad(C), cpad(OC)
    zp = (1 + L["weight_zero"]) if u8 else 0
    if L["op"] == abi.OP_FC:
        return dict(kind="gemm", **gemm_geometry(ocp, zp, m=n, k=Hh * W * cp))
    kind = conv_kind(g, L)
    if kind == "gemm":
        return dict(kind=kind, **gemm_geometry(ocp, zp, m=n * Hh * W, k=cp))
    if kind == "igemm":
        return dict(kind=kind, **gemm_geometry(ocp, zp, conv=dict(n=n, h=Hh, w=W, cp=cp, oh=OH, ow=OW, kh=L["kernel_h"],
                                                                   kw=L["kernel_w"], stride=L["stride_h"], ph0=L["pad_h0"],
                                                                   pw0=L["pad_w0"])))
    if kind == "dw":
        D = dw_geometry(u8, L["kernel_h"], L["kernel_w"], L["stride_h"] if L["stride_h"] == L["stride_w"] else 0, OH, OW,
                        max(L["dilation_h"], L["dilation_w"]))
        return dict(kind=kind, cp_mod32=cp % 32, **D)
    return dict(kind=kind)


KERNEL_NAME = {"gemm": "gemm_i8_tcgen05", "igemm": "conv_igemm_i8_tcgen05", "direct": "conv_direct_dp4a"}  # engine.cu kStepName


def kernel_name(geo):
    if geo["kind"] == "dw":
        return "conv_dw3x3_tma_dp4a" if geo["valid"] else "conv_dw_direct"  # engine.cu:1653
    return KERNEL_NAME[geo["kind"]]


# ---- pooling windows: what makes a window generic ------------------------------------------------------------------------
def pool_geometry(g, L):
    _, _, Hh, W = g.tensors[L["inputs"][0]]["dims"]
    _, _, OH, OW = g.tensors[L["output"]]["dims"]
    wins = ties._pool_windows(dict(L, caffe_flavor=1), Hh, W, OH, OW)
    wins0 = ties._pool_windows(dict(L, caffe_flavor=0), Hh, W, OH, OW)
    return dict(kind="pool",
                square=L["kernel_h"] == L["kernel_w"],
                stride_is_kernel=(L["stride_h"], L["stride_w"]) == (L["kernel_h"], L["kernel_w"]),
                divisors_differ=any(a[-1] != b[-1] for a, b in zip(wins, wins0)),
                one_sided_pad=(L["pad_h0"] > 0) != (L["pad_h1"] > 0) or (L["pad_w0"] > 0) != (L["pad_w1"] > 0))


def geometry(g, L):
    if L["op"] in (abi.OP_CONV, abi.OP_FC):
        return layer_geometry(g, L)
    if L["op"] == abi.OP_POOL:
        return pool_geometry(g, L)
    if L["op"] == abi.OP_CONCAT:
        # engine.cu concat step: an input takes the byte table when its channel count and channel offset are multiples of 16
        offs = np.cumsum([0] + [g.tensors[t]["dims"][1] for t in L["inputs"]])
        table = [g.tensors[t]["dims"][1] % 16 == 0 and o % 16 == 0 for t, o in zip(L["inputs"], offs)]
        return dict(kind="concat", inputs=len(table), mixed=any(table) and not all(table))
    C = g.tensors[L["inputs"][0]]["dims"][1]
    return dict(kind=abi.OP_NAMES[L["op"]], c_mod16=C % 16, channels=C)


# ---- the table ------------------------------------------------------------------------------------------------------------
@dataclass
class Entry:
    name: str
    build: object          # rng -> ties.Case
    kernel: str            # what tb200_graph_layer_kernel reports for the layer under test
    edges: dict            # geometry the entry is meant to reach: key of geometry() -> value
    layer: int = 0         # index of the layer under test
    tie_layer: int = -1    # index of the layer whose rounding is tie-dense (fused pairs: the first)
    ref: str = "exact"     # "exact": ties.exact_run; "oracle": the oracle (ops outside ties.exact_layer)
    fused: bool = False    # run under the default plan (node fusion on); only the graph output is compared
    ties: bool = True      # built tie-dense (ties.check_not_vacuous applies)
    notes: dict = field(default_factory=dict)


ENTRIES = {}


def _add(name, build, kernel, edges, **kw):
    assert name not in ENTRIES, name
    ENTRIES[name] = Entry(name, build, kernel, edges, **kw)


def _rng(name):
    return np.random.default_rng(sum(name.encode()) * 104729)


def build(name):
    e = ENTRIES[name]
    case = e.build(_rng(name))
    case.name = name
    return case


def _i8(*a, **k):
    return lambda r: ties.int8_conv(r, *a, **k)


def _u8(*a, **k):
    return lambda r: ties.uint8_conv(r, *a, **k)


def int8_fc_hw(rng, n, c, h, w, oc, mode=0, m_exps=ties.M_EXPS, tie_frac=0.10):
    """int8 FC over an [n, c, h, w] input (K = c*h*w; the device pads every pixel's channels to 16, so with c % 16 != 0 the pad
    lanes lie inside K).  As ties.int8_fc: roundf(acc * rq), mode 2 through a hot channel."""
    g = GraphDef(abi.DT_INT8)
    x = g.input(n, c, h, w, ties.S_IN)
    k = c * h * w
    wq, ws, m = ties._int8_weights(rng, oc, (k,), k, m_exps)
    if mode == 2:
        m[0] = 1
        ws[0] = 2.0 ** -3
        wq[0] = rng.choice(np.array([-127, 127], np.int8), k)
    b = ties._int8_bias(rng, oc, m, 1)
    g.mark_output(g.fc(x, wq, b, ws, ties.S_OUT))
    xin = rng.integers(-ties.X_MAX, ties.X_MAX + 1, (n, c, h, w)).astype(np.int8)
    cs = ties.Case(f"int8_fc_n{n}c{c}_{h}x{w}_oc{oc}_m{mode}", g, [xin], min_tie_frac=tie_frac)
    cs.mode = ties.planned_mode(g, g.layers[0])
    assert cs.mode == mode, (cs.name, cs.mode)
    return cs


def u8_conv_pad(rng, n, c, h, w, oc, k, stride, pad, mode=0):
    """uint8 conv with a 4-tuple padding (h0, h1, w0, w1): ties.uint8_conv's layer, rebuilt through g.conv(..., pad=...)."""
    case = ties.uint8_conv(rng, n, c, h, w, oc, k=k, stride=stride, pad=0, mode=mode)
    return _repad(case, pad)


def i8_conv_pad(rng, n, c, h, w, oc, k, stride, pad, mode=1):
    case = ties.int8_conv(rng, n, c, h, w, oc, k=k, stride=stride, pad=0, mode=mode)
    return _repad(case, pad)


def _repad(case, pad):
    g0 = case.g
    L = g0.layers[0]
    t0, to = g0.tensors[L["inputs"][0]], g0.tensors[L["output"]]
    g = GraphDef(g0.data_type)
    x = g.input(*t0["dims"], t0["scale"], t0["zero_point"])
    y = g.conv(x, L["weight"], L["bias"], L["weight_scales"], to["scale"], to["zero_point"], stride=L["stride_h"], pad=pad,
               group=L["group"], activation=L["activation"], recipe=L["recipe"], weight_zero=L["weight_zero"])
    g.mark_output(y)
    case.g = g
    case.mode = ties.planned_mode(g, g.layers[0])
    return case


def concat_n(rng, u8, chans, shape=(2, 5, 7)):
    """Concat of len(chans) inputs with s_in / s_out = 1/2, 1/4, 1/2, ... (t = q/2, q/4): inputs whose channel count and offset
    are multiples of 16 take the byte table, the others the bytewise path (engine.cu concat step)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    n, h, w = shape
    ins, xs = [], []
    for i, c in enumerate(chans):
        zp = (120 + 5 * i) if u8 else 0
        ins.append(g.input(n, c, h, w, 2.0 ** -(5 + i % 2), zp))
        xs.append(ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zp))
    g.mark_output(g.concat(ins, 2.0 ** -4, 110 if u8 else 0))
    return ties.Case(("uint8" if u8 else "int8") + "_concat_" + "_".join(map(str, chans)), g, xs, min_tie_frac=0.10)


def relu_maxpool(rng, u8, c, slope_exp=None, shape=(2, 9, 11)):
    """(Leaky) ReLU, then a 3x3 / 2 max pooling keeping the ReLU's quantisation: the pooling folds the ReLU in as a byte table
    (engine.cu fuse_nodes) when the ReLU's output is read by the pooling alone."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi, zo = (128, 110) if u8 else (0, 0)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -5, zi)
    y = g.relu(x, 2.0 ** -4, zo, negative_slope=0.0 if slope_exp is None else 2.0 ** -slope_exp)
    g.mark_output(g.pool(y, abi.POOL_MAX, 3, 2, 1))
    xs = [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zi)]
    return ties.Case(("uint8" if u8 else "int8") + f"_relu_maxpool_c{c}", g, xs, min_tie_frac=0.20)


def eltwise_relu(rng, u8, c, shape=(2, 9, 11)):
    """Eltwise SUM, then a ReLU with the sum's own quantisation: folded into the eltwise kernel (engine.cu fuse_nodes)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    z0, z1, zo = (120, 130, 110) if u8 else (0, 0, 0)
    n, h, w = shape
    a = g.input(n, c, h, w, 2.0 ** -4, z0)
    b = g.input(n, c, h, w, 2.0 ** -5, z1)
    s = g.eltwise(a, b, 2.0 ** -4, zo, elt_type=abi.ELT_SUM)
    g.mark_output(g.relu(s))
    xs = [ties._in(rng, u8, (n, c, h, w), -60, 60, zp=z0), ties._in(rng, u8, (n, c, h, w), -60, 60, zp=z1)]
    return ties.Case(("uint8" if u8 else "int8") + f"_eltwise_relu_c{c}", g, xs, min_tie_frac=0.05)


def silu(rng, c, shape=(2, 9, 11)):
    """x * sigmoid(x) (int8 YOLOv5s' SiLU): the pair becomes one byte table (engine.cu fuse_nodes)."""
    g = GraphDef(abi.DT_INT8)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -4)
    s = g.sigmoid(x, 2.0 ** -7)
    g.mark_output(g.eltwise(x, s, 2.0 ** -4, elt_type=abi.ELT_PROD))
    return ties.Case(f"int8_silu_c{c}", g, [ties._in(rng, False, (n, c, h, w), -127, 127)])


def softmax(rng, u8, c, h=1, w=1, n=3):
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi = 128 if u8 else 0
    x = g.input(n, c, h, w, 2.0 ** -4, zi)
    g.mark_output(g.softmax(x, 2.0 ** -7 if not u8 else 2.0 ** -8, 0))
    return ties.Case(("uint8" if u8 else "int8") + f"_softmax_c{c}_{h}x{w}", g, [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zi)])


def upsample(rng, u8, c, scale, shape=(2, 5, 6)):
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -4, 128 if u8 else 0)
    g.mark_output(g.upsample(x, scale))
    return ties.Case(("uint8" if u8 else "int8") + f"_upsample{scale}_c{c}", g, [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=128 if u8 else 0)])


G_, I_, D_, DD = "gemm_i8_tcgen05", "conv_igemm_i8_tcgen05", "conv_dw3x3_tma_dp4a", "conv_dw_direct"
LOW_M = (2, 2, 3, 4, 5)  # M_c >= 2^-2: the fast-path proof holds up to K ~ 1000

# ---- flat GEMM ------------------------------------------------------------------------------------------------------------
# epilogue constants reloaded per N tile (par_all 0) past PAR_MAX = 2048 channels, resident up to it
_add("gemm1x1_i8_ocp2048", _i8(1, 64, 4, 4, 2048, mode=1), G_, dict(par_all=1, n_tiles=16))
_add("gemm1x1_i8_ocp2064", _i8(1, 64, 4, 4, 2064, mode=1), G_, dict(par_all=0, n_tiles=17))
_add("gemm1x1_u8_ocp2560", _u8(1, 64, 4, 4, 2560), G_, dict(par_all=0))
_add("fc_i8_oc4096", lambda r: ties.int8_fc(r, 2, 256, 4096), G_, dict(par_all=0, n_tiles=32))
# uneven N tiles: block_n does not divide ocp
for oc, bn in ((144, 80), (272, 96), (400, 112)):
    _add(f"gemm1x1_i8_ocp{oc}", _i8(2, 64, 9, 7, oc, mode=1), G_, dict(n_uneven=True, block_n=bn))
_add("gemm1x1_i8_ocp256", _i8(2, 64, 9, 7, 256, mode=1), G_, dict(n_uneven=False, block_n=128))
_add("gemm1x1_u8_ocp144", _u8(2, 64, 9, 7, 144), G_, dict(n_uneven=True))
# the last m-tile: M % 128 = 1 and 127 (and 0)
_add("gemm1x1_i8_m129", _i8(1, 64, 3, 43, 40, mode=1), G_, dict(m_rem=1))
_add("gemm1x1_i8_m255", _i8(1, 64, 5, 51, 40, mode=0), G_, dict(m_rem=127))
_add("gemm1x1_i8_m256", _i8(1, 64, 8, 32, 40, mode=1), G_, dict(m_rem=0))
_add("gemm1x1_u8_m129", _u8(1, 64, 3, 43, 40), G_, dict(m_rem=1))
# m-tiles per accumulator stage: 1 (128-channel tile), 2 (64 channels), 4 (32 channels, >= 4 m-tiles); 32 channels over 3 m-tiles: 2
_add("gemm1x1_i8_mt1", _i8(2, 64, 15, 20, 125, mode=1), G_, dict(mt=1))
_add("gemm1x1_i8_mt2", _i8(2, 64, 15, 20, 64, mode=1), G_, dict(mt=2))
_add("gemm1x1_i8_mt4", _i8(2, 64, 15, 20, 32, mode=0), G_, dict(mt=4, cs=2))
_add("gemm1x1_i8_mt4_3tiles", _i8(1, 64, 16, 24, 32, mode=1), G_, dict(mt=2, m_tiles=3))
_add("gemm1x1_u8_mt4", _u8(2, 64, 15, 20, 32), G_, dict(mt=4))
# FC over an HxW > 1 input with C % 16 != 0: the pad lanes of every pixel lie inside K
_add("fc_i8_c24_3x3", lambda r: int8_fc_hw(r, 3, 24, 3, 3, 50, m_exps=LOW_M), G_, dict(block_k=128, k_blocks=3))
_add("fc_u8_c24_3x3", lambda r: ties.uint8_conv(r, 3, 24, 3, 3, 50, fc=True), G_, dict(block_k=128, k_blocks=3))
# long K (VGG fc6: 512 x 7 x 7 = 25088): 196 k-blocks, weights streamed
_add("fc_i8_vgg_fc6", lambda r: int8_fc_hw(r, 8, 512, 7, 7, 96, mode=2, tie_frac=0.03), G_, dict(k_blocks=196, b_res=0))
_add("fc_i8_k1024_resident", lambda r: int8_fc_hw(r, 2, 64, 4, 4, 96, mode=2), G_, dict(k_blocks=8, b_res=1))
_add("fc_u8_vgg_fc6", lambda r: ties.uint8_conv(r, 2, 512, 7, 7, 64, fc=True, mode=2), G_, dict(k_blocks=196, b_res=0))

# ---- implicit GEMM ---------------------------------------------------------------------------------------------------------
# out_mode 1 / 2 exactly at ow 128 / 129
_add("igemm3x3_i8_ow128", _i8(1, 64, 3, 128, 40, k=3, pad=1, mode=1), I_, dict(out_mode=1, bw=128))
_add("igemm3x3_i8_ow129", _i8(1, 64, 3, 129, 40, k=3, pad=1, mode=1), I_, dict(out_mode=2, bw=128))
_add("igemm3x3_u8_ow129", _u8(1, 64, 3, 129, 40, k=3, pad=1), I_, dict(out_mode=2))
# whole-image patches with a partial last m-tile (n % bn != 0), and oh % bh != 0
_add("igemm3x3_i8_bn5_n7", _i8(7, 64, 5, 5, 40, k=3, pad=1, mode=1), I_, dict(out_mode=0, bn=5, n_partial=True, tail=29))
_add("igemm3x3_i8_bn5_n10", _i8(10, 64, 5, 5, 40, k=3, pad=1, mode=1), I_, dict(out_mode=0, bn=5, n_partial=False))
_add("igemm3x3_u8_bn5_n7", _u8(7, 64, 5, 5, 40, k=3, pad=1), I_, dict(out_mode=0, n_partial=True))
_add("igemm3x3_i8_oh15_bh6", _i8(2, 64, 15, 20, 40, k=3, pad=1, mode=1), I_, dict(out_mode=1, bh=6, oh_partial=True, tail=24))
_add("igemm3x3_i8_oh12_bh6", _i8(2, 64, 12, 20, 40, k=3, pad=1, mode=1), I_, dict(out_mode=1, bh=6, oh_partial=False))
# several k-blocks per tap
_add("igemm3x3_i8_cp64", _i8(2, 64, 9, 10, 40, k=3, pad=1, mode=1), I_, dict(block_k=64, cblocks=1))
_add("igemm3x3_i8_cp96", _i8(2, 96, 9, 10, 40, k=3, pad=1, mode=1, m_exps=LOW_M), I_, dict(block_k=32, cblocks=3))
_add("igemm3x3_i8_cp160", _i8(2, 160, 9, 10, 40, k=3, pad=1, mode=2), I_, dict(block_k=32, cblocks=5))
_add("igemm3x3_i8_cp192", _i8(2, 192, 9, 10, 40, k=3, pad=1, mode=2), I_, dict(block_k=64, cblocks=3))
_add("igemm3x3_u8_cp96", _u8(2, 96, 9, 10, 40, k=3, pad=1, mode=2), I_, dict(block_k=32, cblocks=3, border=1))
# 5x5 and 7x7 interiors (25 / 49 taps), uint8 border tables with pad 2 / 3
_add("igemm5x5_i8_p2", _i8(2, 64, 11, 12, 40, k=5, pad=2, mode=2), I_, dict(taps=25))
_add("igemm7x7_i8_p3", _i8(1, 64, 13, 12, 40, k=7, pad=3, mode=2), I_, dict(taps=49))
_add("igemm5x5_u8_p2", _u8(2, 64, 11, 12, 40, k=5, pad=2, mode=2), I_, dict(taps=25, border=1))
_add("igemm7x7_u8_p3", _u8(1, 64, 13, 12, 40, k=7, pad=3, mode=2), I_, dict(taps=49, border=1))
# images smaller than the kernel window
_add("igemm5x5_i8_img3x3", _i8(4, 64, 3, 3, 40, k=5, pad=2, mode=2), I_, dict(taps=25, out_mode=0))
_add("igemm7x7_u8_img2x2", _u8(4, 64, 2, 2, 40, k=7, pad=3, mode=2), I_, dict(taps=49, out_mode=0, border=1))
# uneven N tiles through the implicit GEMM
_add("igemm3x3_i8_ocp272", _i8(2, 64, 9, 10, 272, k=3, pad=1, mode=1), I_, dict(n_uneven=True, n_tiles=3))
_add("igemm3x3_u8_ocp400", _u8(2, 64, 9, 10, 400, k=3, pad=1), I_, dict(n_uneven=True, n_tiles=4))
# TF-style asymmetric padding (0, 1) at stride 2; a 1x1 window with it has border pixels only at the bottom / right
_add("igemm3x3s2_i8_pad01", lambda r: i8_conv_pad(r, 2, 64, 24, 30, 40, 3, 2, (0, 1, 0, 1)), I_, dict(out_mode=1))
_add("igemm3x3s2_u8_pad01", lambda r: u8_conv_pad(r, 2, 64, 12, 14, 40, 3, 2, (0, 1, 0, 1)), I_, dict(border=1))
_add("igemm1x1s2_u8_pad01", lambda r: u8_conv_pad(r, 2, 64, 12, 14, 40, 1, 2, (0, 1, 0, 1)), I_, dict(taps=1, border=1))
_add("igemm1x1s1_u8_pad01", lambda r: u8_conv_pad(r, 2, 64, 9, 10, 40, 1, 1, (0, 1, 0, 1)), I_, dict(taps=1, border=1))
_add("igemm1x1s2_u8_nopad", _u8(2, 64, 13, 15, 40, k=1, stride=2), I_, dict(taps=1, border=0))

# ---- depthwise 3x3 -------------------------------------------------------------------------------------------------------
# the last 32-channel chunk half outside the tensor (cp % 32 == 16): MobileNet-v2's 144 channels
_add("dw3x3s1_i8_c144", _i8(2, 144, 13, 14, 144, k=3, pad=1, group=144, mode=1), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s2_i8_c48", _i8(2, 48, 13, 14, 48, k=3, stride=2, pad=1, group=48, mode=0), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s1_i8_c40", _i8(2, 40, 9, 10, 40, k=3, pad=1, group=40, mode=2), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s1_i8_c64", _i8(2, 64, 9, 10, 64, k=3, pad=1, group=64, mode=1), D_, dict(valid=True, cp_mod32=0))
_add("dw3x3s1_u8_c144", _u8(1, 144, 9, 10, 144, k=3, pad=1, group=144), DD, dict(valid=False, cp_mod32=16))
# the row limit: 16 pixel groups (ow 128 at stride 1, 64 at stride 2); one more pixel takes the generic kernel
_add("dw3x3s1_i8_ow128", _i8(1, 48, 4, 128, 48, k=3, pad=1, group=48, mode=1), D_, dict(valid=True, gpr=16, stride=1))
_add("dw3x3s1_i8_ow129", _i8(1, 48, 4, 129, 48, k=3, pad=1, group=48, mode=1), DD, dict(valid=False, gpr=17, stride=1))
_add("dw3x3s2_i8_ow64", _i8(1, 48, 6, 128, 48, k=3, stride=2, pad=1, group=48, mode=1), D_, dict(valid=True, gpr=16, stride=2))
_add("dw3x3s2_i8_ow65", _i8(1, 48, 6, 129, 48, k=3, stride=2, pad=1, group=48, mode=1), DD, dict(valid=False, gpr=17, stride=2))
# fewer output rows than rows_per_cta
_add("dw3x3s1_i8_oh3_capped", _i8(2, 32, 3, 8, 32, k=3, pad=1, group=32, mode=1), D_, dict(valid=True, rows_capped=True, rows_per_cta=3))
_add("dw3x3s1_i8_oh1_capped", _i8(3, 32, 1, 20, 32, k=3, pad=1, group=32, mode=0), D_, dict(valid=True, rows_capped=True, rows_per_cta=1))
_add("dw3x3s2_i8_oh2_capped", _i8(2, 48, 3, 30, 48, k=3, stride=2, pad=1, group=48, mode=1), D_, dict(valid=True, rows_capped=True))
_add("dw3x3s1_i8_oh17_full", _i8(1, 32, 17, 30, 32, k=3, pad=1, group=32, mode=1), D_, dict(valid=True, rows_capped=False, rows_per_cta=4))

# ---- glue ----------------------------------------------------------------------------------------------------------------
_P = "pool"
for d, u in (("i8", False), ("u8", True)):
    # non-square windows, stride != kernel, clipped windows (caffe vs plain divisors), padding on one side only
    _add(f"avgpool2x4s2x4_{d}", lambda r, u=u: ties.pool(r, u, abi.POOL_AVG, (2, 4), (2, 4), shape=(2, 20, 8, 12)), _P,
         dict(square=False, stride_is_kernel=True))
    _add(f"maxpool2x3s1_{d}", lambda r, u=u: ties.pool(r, u, abi.POOL_MAX, (2, 3), 1, scale_ratio=2), _P,
         dict(square=False, stride_is_kernel=False))
    _add(f"avgpool2x2s1_{d}", lambda r, u=u: ties.pool(r, u, abi.POOL_AVG, 2, 1), _P, dict(square=True, stride_is_kernel=False))
    for caffe in (0, 1):
        _add(f"avgpool3x3s2p1_caffe{caffe}_{d}", lambda r, u=u, c=caffe: ties.pool(r, u, abi.POOL_AVG, 3, 2, pad=1, caffe=c,
                                                                                   shape=(2, 20, 9, 10)),
             _P, dict(divisors_differ=True), ref="oracle", ties=False)
        _add(f"avgpool2x2p_top_caffe{caffe}_{d}", lambda r, u=u, c=caffe: ties.pool(r, u, abi.POOL_AVG, 2, 2, pad=(1, 0, 0, 0),
                                                                                    caffe=c, shape=(2, 20, 9, 10)),
             _P, dict(one_sided_pad=True))
    _add(f"maxpool3x3s2_p_left_{d}", lambda r, u=u: ties.pool(r, u, abi.POOL_MAX, 3, 2, pad=(0, 0, 1, 0), scale_ratio=2,
                                                             shape=(2, 20, 9, 10)), _P, dict(one_sided_pad=True))
    _add(f"avgpool2x2s2_{d}", lambda r, u=u: ties.pool(r, u, abi.POOL_AVG, 2, 2), _P,
         dict(one_sided_pad=False, divisors_differ=False, square=True, stride_is_kernel=True))
    # concat of 3 / 4 inputs mixing byte-table (16-aligned channels and offset) and bytewise inputs
    _add(f"concat4_{d}", lambda r, u=u: concat_n(r, u, (16, 8, 24, 16)), "concat_requant", dict(inputs=4, mixed=True))
    _add(f"concat3_{d}", lambda r, u=u: concat_n(r, u, (32, 40, 16)), "concat_requant", dict(inputs=3, mixed=True))
    _add(f"concat3_aligned_{d}", lambda r, u=u: concat_n(r, u, (16, 32, 16)), "concat_requant", dict(inputs=3, mixed=False))
    # upsample x3 at C % 16 != 0
    _add(f"upsample3_c24_{d}", lambda r, u=u: upsample(r, u, 24, 3), "upsample_nearest", dict(c_mod16=8), ref="oracle", ties=False)
    # softmax over 1 and 1000 channels, and per spatial position
    for c, h, w in ((1, 1, 1), (1000, 1, 1), (21, 5, 6)):
        _add(f"softmax_c{c}_{h}x{w}_{d}", lambda r, u=u, c=c, h=h, w=w: softmax(r, u, c, h, w), "softmax", dict(channels=c),
             ref="oracle", ties=False)
_add("upsample3_c32_i8", lambda r: upsample(r, False, 32, 3), "upsample_nearest", dict(c_mod16=0), ref="oracle", ties=False)

# fused paths (default plan; the fused tensor is the graph output)
_F = "fused_into_producer"
_add("relu_maxpool_u8_c24", lambda r: relu_maxpool(r, True, 24), _F, dict(c_mod16=8), fused=True, tie_layer=0)
_add("relu_maxpool_u8_c32", lambda r: relu_maxpool(r, True, 32), _F, dict(c_mod16=0), fused=True, tie_layer=0)
_add("leaky_relu_maxpool_i8_c24", lambda r: relu_maxpool(r, False, 24, slope_exp=2), _F, dict(c_mod16=8), fused=True, tie_layer=0)
_add("eltwise_relu_i8_c24", lambda r: eltwise_relu(r, False, 24), _F, dict(c_mod16=8), layer=1, fused=True, tie_layer=0)
_add("eltwise_relu_u8_c32", lambda r: eltwise_relu(r, True, 32), _F, dict(c_mod16=0), layer=1, fused=True, tie_layer=0)
_add("silu_i8_c24", lambda r: silu(r, 24), _F, dict(c_mod16=8), fused=True, ref="oracle", ties=False)

# Boundaries: geometry key -> the values that must each be reached by some entry (both sides of every edge)
BOUNDARIES = {
    "par_all": {0, 1},
    "n_uneven": {True, False},
    "m_rem": {0, 1, 127},
    "mt": {1, 2, 4},
    "b_res": {0, 1},
    "out_mode": {0, 1, 2},
    "n_partial": {True, False},
    "oh_partial": {True, False},
    "cblocks": {1, 3, 5},
    "taps": {1, 25, 49},
    "border": {0, 1},
    "valid": {True, False},
    "gpr": {16, 17},
    "cp_mod32": {0, 16},
    "rows_capped": {True, False},
    "square": {True, False},
    "stride_is_kernel": {True, False},
    "divisors_differ": {True, False},
    "one_sided_pad": {True, False},
    "c_mod16": {0, 8},
    "mixed": {True, False},
}

# Edges no graph can reach, and why (none so far).
UNREACHABLE = {}


def gemm_entries():
    return [n for n, e in ENTRIES.items() if e.kernel in (G_, I_)]


def uint8_gemm_entries():
    return [n for n in gemm_entries() if "_u8_" in n or n.startswith("fc_u8")]

