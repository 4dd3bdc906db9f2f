"""Single-layer cases at the edges of each kernel's tiling and of the planner's kernel choice, with the host-side plan geometry
restated in Python.

The tie-dense builders of tests/ties.py make the layers (power-of-two scales: `ties.exact_run` is an exact reference, independent
of the oracle); ops that `ties.exact_layer` does not cover (softmax, upsample, sigmoid) are compared with the oracle instead.

`gemm_geometry`, `dw_geometry`, `window_geometry`, `gather_geometry`, `epi_clamp` and `conv_kind` restate the C planners line by
line (cited at each function).  They only describe what the library decides -- no plan logic lives here -- so that the CPU test
can show every entry reaches the geometry it is meant to, and the GPU test can tie the restatement to the library
(TB200_DEBUG_LAUNCH prints the plans of the GEMM, the window and the gather kernel).  `conv_recipe` restates the device glue's
choice of float recipe, the one the unmodified reference would run: every conv entry has it, or is marked `abi_only`.

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
PLAN_STG_WARPS, SMEM_CTL = 16, 432  # sizeof(GemmSmemCtl): (2 * MAX_STAGES + 5) uint64, 16-byte aligned


def _block_n(ocp):
    nt = (ocp + 127) // 128  # gemm_block_n
    return ((ocp + nt - 1) // nt + 15) & ~15


def gemm_geometry(ocp, u8zp, m=None, k=None, conv=None):
    """The plan of gemm_plan_create (flat: m rows, k = K) or gemm_plan_create_conv (conv = dict(n, h, w, cp, oh, ow, kh, kw,
    stride, ph0, pw0)).  u8zp is the planners' `u8` argument: 0 for int8, 1 + weight zero point for uint8.  Restates
    gemm_tcgen05.cu gemm_block_n, plan_begin, gemm_plan_create, gemm_plan_create_conv (with its BORDER), plan_stage, and
    plan_ring with epilogue_smem_bytes (par_all, b_res)."""
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
    # plan_begin: uint8 B holds w - 128 (signed) unless zw == 0, and the epilogue adds cplane * sum(x) with cplane = 128 - zw;
    # gemm_mma_dispatch<AU, BU = !b_signed> picks the MMA warpgroup's code by (block_n, mt)
    G["b_signed"] = int(u8zp != 1)
    G["cplane"] = cplane = 128 - (u8zp - 1) if u8zp > 1 else 0
    if u8zp:
        G["u8_operands"] = {1: "unsigned_b", 129: "no_cplane", 2: "cplane_max", 256: "cplane_min"}.get(u8zp, "cplane")
        G["mma_uu"] = (bn, mt) if u8zp == 1 else None
    epi = PLAN_STG_WARPS * 2 * 512 * cs + (par_ch if par_ch <= PAR_MAX else bn) * 8 + SMEM_CTL + 2048 + 128 * (mt * bn * 4 + 16) + 16
    budget = 224 * 1024 - epi - (4096 if cplane else 0)  # the row sums' region exists only with cplane != 0
    a_bytes, b_al = BLOCK_M * bk, (bn * bk + 1023) & ~1023
    b_res = 1 if kb * b_al <= B_RESIDENT_MAX else 0
    if b_res and (budget - kb * b_al) // a_bytes < 3:
        b_res = 0
    G["b_res"] = b_res
    return G


# ---- dw_tma.cu dw_plan_create: the TMA depthwise 3x3 or the generic kernel ---------------------------------------------------
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


# ---- conv_window.cu: the window kernel's plan and the gather kernel's tiles ---------------------------------------------------
WINDOW_SMEM_MAX = 200 * 1024


def _acc_pitch(ocp):
    return ocp * 4 + 16  # tc_common.cuh acc_pitch


def window_smem_bytes(ks, ocp, in_bytes):
    return ks * 4096 + ks * ocp * 32 + ocp * 8 + 128 + 2 * ((in_bytes + 127) & ~127) + 128 * _acc_pitch(ocp) + 1024


def window_nhwc_fits(cp, ocp, stride):
    box_w, box_h = 15 * stride + 3, 7 * stride + 3
    return window_smem_bytes((9 * cp + 31) // 32, ocp, box_w * box_h * cp) <= WINDOW_SMEM_MAX


def window_geometry(n, c, cp, w, oh, ow, k, stride, pw0, ocp, nhwc):
    """window_plan_create's checks beyond plan_conv's (group 1, no dilation, one stride, square kernel), its box and shared
    memory, and its tiles: 16 x 8 output pixels per tile, the two tile counts divided by
    multiply-high with a magic number, 0 for a divisor of 1."""
    W = dict(valid=False, layout=None)
    if stride > 2 or ocp > 256:
        return W
    if nhwc:
        if k != 3 or cp not in (16, 32):
            return W
        layout, xoff = (2 if cp == 16 else 3), 0
        box_w, box_h = 15 * stride + 3, 7 * stride + 3
        in_bytes, ks = box_w * box_h * cp, (9 * cp + 31) // 32
    else:
        if k not in (3, 7) or c > 3 or w % 16:
            return W
        layout, xoff = (0 if k == 3 else 1), (16 - pw0 % 16) % 16
        box_w, box_h = (xoff + 15 * stride + k + 15) & ~15, 7 * stride + k
        if box_w > 256 or box_h > 256:
            return W
        in_bytes, ks = box_w * box_h * c, (c * k * k + 31) // 32
    W.update(layout=layout, xoff=xoff, box_w=box_w, box_h=box_h, ks=ks, smem_bytes=window_smem_bytes(ks, ocp, in_bytes))
    if W["smem_bytes"] > WINDOW_SMEM_MAX:
        return W
    W["valid"] = True
    W["tiles_w"], W["tiles_h"] = tw, th = (ow + 15) // 16, (oh + 7) // 8
    W["ntiles"] = tw * th * n
    W["tw_magic0"], W["th_magic0"], W["batch1"] = tw == 1, th == 1, n == 1
    W["ow_mod16"], W["oh_mod8"] = ow % 16, oh % 8
    return W


def gather_geometry(n, c, oh, ow, k, nhwc16):
    """gather_plan_create: 128 output pixels per tile; ks k-steps of 32 bytes (NHWC16: nine 16-byte taps and a zero half)."""
    npix = n * oh * ow
    return dict(ks=5 if nhwc16 else (c * k * k + 31) // 32, ntiles=(npix + 127) // 128, npix_mod128=npix % 128)


# ---- engine.cu make_epi: the activation's clamp in the fast epilogues -------------------------------------------------------
def epi_clamp(g, L):
    """The activation's bounds in real units (flo, fhi), over s_out: whether one is a half-integer (the reference rounds the
    clipped value, away from zero), and whether one lies beyond the byte range (the integer clamp is then saturation's)."""
    fc = L["op"] == abi.OP_FC
    act = -1 if fc else L["activation"]
    flo, fhi = -np.inf, np.inf
    if L["recipe"] == abi.RECIPE_HCL or fc:
        if act == 0:
            flo = 0.0
        if act > 0:
            flo, fhi = 0.0, 6.0
    elif act >= 0:
        flo, fhi = (-1.0, 1.0) if act == 1 else (0.0, 6.0 if act == 6 else np.inf)
    tout = g.tensors[L["output"]]
    so, zo = np.float32(tout["scale"]), tout["zero_point"]
    bounds = [b / so for b in (flo, fhi) if np.isfinite(b)]
    lo, hi = (-zo, 255 - zo) if g.data_type == abi.DT_UINT8 else (-127, 127)
    name = "none" if act < 0 else ("hcl" if L["recipe"] == abi.RECIPE_HCL else "ref") + str(act)
    return dict(act=name, bound_half=any(b - np.floor(b) == 0.5 for b in bounds),
                bound_beyond_sat=any(ties._round_away(b) < lo or ties._round_away(b) > hi for b in bounds))


# ---- b200_device.cc conv_recipe: the recipe Tengine's CPU device would run a convolution with ---------------------------------
def conv_recipe(g, L):
    """Group 1: HCL (conv_hcl_x86 / conv_direct_hcl_int8_x86).  A depthwise conv: HCL only for int8 at batch 1, 3x3, one stride of
    1 or 2, no dilation and each axis padded alike on both sides (conv_dw_hcl_x86.c:508-543); every other grouped conv, and every
    uint8 depthwise, runs conv_ref: REF.  A layer with the other recipe can only come from a C-ABI caller."""
    n, C = g.tensors[L["inputs"][0]]["dims"][:2]
    OC = g.tensors[L["output"]]["dims"][1]
    grp = L["group"]
    if grp == 1:
        return abi.RECIPE_HCL
    dw = grp == C and grp == OC
    if (dw and g.data_type == abi.DT_INT8 and n == 1 and L["kernel_h"] == 3 and L["kernel_w"] == 3 and L["stride_h"] == L["stride_w"]
            and L["stride_h"] in (1, 2) and L["dilation_h"] == 1 and L["dilation_w"] == 1 and L["pad_h0"] == L["pad_h1"]
            and L["pad_w0"] == L["pad_w1"]):
        return abi.RECIPE_HCL
    return abi.RECIPE_REF


# ---- engine.cu plan_conv and fill_conv_step: the kernel of a convolution ----------------------------------------------------
def _window_of(g, L, nhwc):
    n, C, _, W = g.tensors[L["inputs"][0]]["dims"]
    _, OC, OH, OW = g.tensors[L["output"]]["dims"]
    return window_geometry(n, C, cpad(C), W, OH, OW, L["kernel_h"], L["stride_h"], L["pad_w0"], cpad(OC), nhwc)


def conv_kind(g, L, no_tc=False):
    """'gemm', 'igemm', 'dw', 'direct', 'stem', 'window' or 'gather'.  plan_conv's K_GATHER_TC (NCHW stem, 16-channel input)
    becomes 'window' when window_plan_create makes a plan, else 'gather' (fill_conv_step); its 32-channel branch needs
    window_nhwc_fits and otherwise falls through to the implicit GEMM."""
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
        return "window" if _window_of(g, L, 0)["valid"] else "gather"
    if is_input and C <= 4 and grp == 1:
        return "stem"
    if gather and k3 and cp == 16:
        return "window" if _window_of(g, L, 1)["valid"] else "gather"
    if gather and k3 and cp == 32 and sh in (1, 2) and window_nhwc_fits(32, ocp, sh):
        return "window"
    if grp == C and OC == C and C > 1:
        return "dw"
    if tc and kh == 1 and kw == 1 and sh == 1 and sw == 1 and nopad:
        return "gemm"
    if tc and plain and sh in (1, 2) and (kh * kw == 1 or cp % 32 == 0) and OW <= 4096 and kh * kw <= 64:
        return "igemm"
    return "direct"


def layer_geometry(g, L, no_tc=False):
    """The restated plan of a conv / FC layer: dict with 'kind', the kind's geometry and the epilogue's clamp."""
    u8 = g.data_type == abi.DT_UINT8
    n, C, Hh, W = g.tensors[L["inputs"][0]]["dims"]
    _, OC, OH, OW = g.tensors[L["output"]]["dims"]
    cp, ocp = cpad(C), cpad(OC)
    zp = (1 + L["weight_zero"]) if u8 else 0
    epi = epi_clamp(g, L)
    if L["op"] == abi.OP_FC:
        if no_tc:
            return dict(kind="direct", oct=8, **epi)
        return dict(kind="gemm", **gemm_geometry(ocp, zp, m=n, k=Hh * W * cp), **epi)
    kind = conv_kind(g, L, no_tc)
    if kind == "gemm":
        return dict(kind=kind, **gemm_geometry(ocp, zp, m=n * Hh * W, k=cp), **epi)
    if kind == "igemm":
        return dict(kind=kind, **gemm_geometry(ocp, zp, conv=dict(n=n, h=Hh, w=W, cp=cp, oh=OH, ow=OW, kh=L["kernel_h"],
                                                                   kw=L["kernel_w"], stride=L["stride_h"], ph0=L["pad_h0"],
                                                                   pw0=L["pad_w0"])), **epi)
    if kind == "dw":
        s = L["stride_h"] if L["stride_h"] == L["stride_w"] else 0
        D = dw_geometry(u8, L["kernel_h"], L["kernel_w"], s, OH, OW, max(L["dilation_h"], L["dilation_w"]))
        if no_tc:
            D["valid"] = False  # fill_conv_step makes no TMA plan
        # kernels_direct.cu launch_conv_dw without a TMA plan: int8 3x3 at stride 1 / 2 takes TW output pixels per thread
        i8_3x3 = not u8 and L["kernel_h"] == L["kernel_w"] == 3 and max(L["dilation_h"], L["dilation_w"]) == 1 and s in (1, 2)
        if not D["valid"]:
            D["dw_kernel"] = "dw3x3_i8" if i8_3x3 else "generic"
            D["dw_ow_tail"] = OW % (8 if s == 1 else 4) if i8_3x3 else None
        return dict(kind=kind, cp_mod32=cp % 32, **D, **epi)
    nhwc = cp in (16, 32) and not (C <= 3 and L["inputs"][0] in g.inputs)
    if kind == "window":
        return dict(kind=kind, window_valid=True, **_window_of(g, L, int(nhwc)), **epi)
    if kind == "gather":
        return dict(kind=kind, window_valid=False, **gather_geometry(n, C, OH, OW, L["kernel_h"], int(nhwc)), **epi)
    if kind == "stem":
        return dict(kind=kind, oct=32 if ocp % 32 == 0 else 16, **epi)  # kernels_direct.cu launch_conv_stem
    og = OC // L["group"]
    return dict(kind=kind, oct=4 if L["group"] > 1 and og % 8 else 8, **epi)  # kernels_direct.cu launch_conv_direct


# engine.cu kStepName, per step kind
KERNEL_NAME = {"gemm": "gemm_i8_tcgen05", "igemm": "conv_igemm_i8_tcgen05", "direct": "conv_direct_dp4a", "stem": "conv_stem_nchw_dp4a",
               "window": "conv_window_tcgen05", "gather": "conv_gather_tcgen05"}


def kernel_name(geo):
    if geo["kind"] == "dw":
        return "conv_dw3x3_tma_dp4a" if geo["valid"] else "conv_dw_direct"  # engine.cu fill_conv_step: K_CONV_DW_TMA or K_CONV_DW
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


def geometry(g, L, no_tc=False):
    if L["op"] in (abi.OP_CONV, abi.OP_FC):
        return layer_geometry(g, L, no_tc)
    if L["op"] == abi.OP_POOL:
        return pool_geometry(g, L)
    if L["op"] == abi.OP_CONCAT:
        # engine.cu fill_concat_steps: an input takes the byte table (K_CONCAT_LUT) when its channel count and offset are multiples of 16
        offs = np.cumsum([0] + [g.tensors[t]["dims"][1] for t in L["inputs"]])
        table = [g.tensors[t]["dims"][1] % 16 == 0 and o % 16 == 0 for t, o in zip(L["inputs"], offs)]
        return dict(kind="concat", inputs=len(table), mixed=any(table) and not all(table))
    C = g.tensors[L["inputs"][0]]["dims"][1]
    return dict(kind=abi.OP_NAMES[L["op"]], c_mod16=C % 16, channels=C)


def data_edges(case, e):
    """What an entry's quantisation and data reach beyond the plan: uint8 input and output zero points (zx, zo), whether a uint8
    pooling result falls below 0 and wraps (pool_wraps), and whether an int8 graph input holds -128 (in_min_byte)."""
    g = case.g
    L = g.layers[e.layer]
    if g.data_type != abi.DT_UINT8:
        return dict(in_min_byte=any(bool((np.asarray(x) == -128).any()) for x in case.inputs))
    D = dict(zx=g.tensors[L["inputs"][0]]["zero_point"], zo=g.tensors[L["output"]]["zero_point"])
    if L["op"] == abi.OP_POOL and e.ref == "exact":
        r = ties.exact_run(g, case.inputs)[1][L["output"]]
        D["pool_wraps"] = bool((ties._round_away(r.t) + r.add < 0).any())
    return D


def reached(case, e):
    """geometry() of the entry's layer and its data_edges."""
    no_tc = bool(e.flags & abi.PRERUN_NO_TENSORCORE)
    return dict(geometry(case.g, case.g.layers[e.layer], no_tc=no_tc), **data_edges(case, e))


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
    flags: int = 0         # prerun flags ORed into the run's (PRERUN_NO_TENSORCORE: the CUDA-core kernels)
    abi_only: bool = False  # a conv whose recipe is not conv_recipe's for its shape: only a C-ABI caller can ask for it, so the
    #                         unmodified reference (which picks its own) is no judge of it: not run through it
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


def u8_conv_pad(rng, n, c, h, w, oc, k, stride, pad, mode=0, dilation=1, **zps):
    """uint8 conv with a 4-tuple padding (h0, h1, w0, w1) or a dilation: ties.uint8_conv's layer, rebuilt through
    g.conv(..., pad=..., dilation=...).  zps: ties.uint8_conv's zero points."""
    case = ties.uint8_conv(rng, n, c, h, w, oc, k=k, stride=stride, pad=0, mode=mode, **zps)
    return _repad(case, pad, dilation)


def u8_far(rng, n, c, h, w, oc, k=1, pad=0, fc=False, zx=255, zw=0, s_out=16.0):
    """uint8 conv / FC with inputs and weights at the far ends of the byte range from their zero points (|x - zx| and |w - zw| in
    [235, 255]), so that the accumulator nears 255^2 K (1.6e9 at K = 25088, 3/4 of int32).  The bias takes each channel's median
    accumulator off (padded: the interior's) and s_out spreads t over about +-40.  Past 2^24 the reference rounds the accumulator
    to fp32 before it scales it, which ties.exact_layer does not model: compared with the oracle.  MODE 2 (the clamp-range proof
    fails)."""
    g = GraphDef(abi.DT_UINT8)
    s_in, s_w = 2.0 ** -4, 2.0 ** -3
    x = g.input(n, c, h, w, s_in, zx)
    kk = c * h * w if fc else c * k * k
    far = lambda z, shape: ((0 if z > 127 else 235) + rng.integers(0, 21, shape)).astype(np.uint8)  # noqa: E731
    wq = far(zw, (oc, kk) if fc else (oc, c, k, k))
    xin = far(zx, (n, c, h, w))
    L = dict(group=1, stride_h=1, stride_w=1, dilation_h=1, dilation_w=1, pad_h0=pad, pad_h1=pad, pad_w0=pad, pad_w1=pad)
    acc = ties.conv_acc(xin.reshape(n, 1, 1, -1), wq.reshape(oc, 1, 1, -1), dict(L, pad_h0=0, pad_h1=0, pad_w0=0, pad_w1=0), zx, zw) \
        if fc else ties.conv_acc(xin, wq, L, zx, zw)
    b = (-np.rint(np.median(acc, axis=(0, 2, 3))) + rng.integers(-40, 41, oc) * s_out / (s_in * s_w)).astype(np.int32)
    if fc:
        y = g.fc(x, wq, b, [s_w], s_out, 128, weight_zero=zw)
    else:
        y = g.conv(x, wq, b, [s_w], s_out, 128, pad=pad, weight_zero=zw)
    g.mark_output(y)
    cs = ties.Case(f"uint8_far_{'fc' if fc else f'k{k}'}_K{kk}_z{zx}_{zw}", g, [xin])
    cs.mode = ties.planned_mode(g, g.layers[0])
    cs.notes["acc_max"] = int(np.abs(acc).max())
    assert cs.mode == 2, cs.name
    return cs


def i8_conv_pad(rng, n, c, h, w, oc, k, stride, pad, mode=1, dilation=1):
    case = ties.int8_conv(rng, n, c, h, w, oc, k=k, stride=stride, pad=0, mode=mode)
    return _repad(case, pad, dilation)


def _repad(case, pad, dilation=1):
    g0 = case.g
    L = g0.layers[0]
    t0, to = g0.tensors[L["inputs"][0]], g0.tensors[L["output"]]
    g = GraphDef(g0.data_type)
    x = g.input(*t0["dims"], t0["scale"], t0["zero_point"])
    y = g.conv(x, L["weight"], L["bias"], L["weight_scales"], to["scale"], to["zero_point"], stride=L["stride_h"], pad=pad,
               dilation=dilation, group=L["group"], activation=L["activation"], recipe=L["recipe"], weight_zero=L["weight_zero"])
    g.mark_output(y)
    case.g = g
    case.mode = ties.planned_mode(g, g.layers[0])
    return case


def act_conv(rng, u8, n, c, h, w, oc, activation, recipe, s_out, k=3, stride=1, pad=1, group=1, zo=110, t_mid=0.0, zx=ties.U8_ZX,
             zw=ties.U8_ZW, min_byte=False):
    """A conv whose t = f / s_out lies within a few units of t_mid, so that the activation's clamp cuts it: the clamp bounds over
    a power-of-two s_out (6 / 4 = 1.5, 1 / 2 = 0.5) are half-integers, which the reference rounds away from zero.  M = 2^-1
    (every odd accumulator is a tie); weights +-1 on about six taps per output, inputs in [-2, 2] about the zero point, so t
    spreads over about +-2 whatever K is.  uint8 zero points zx, zw, zo: at an end of the byte range the inputs are
    [0, 4] or [251, 255] (ties._shift) and the weights zw + {0, 1} or zw - {0, 1}; the bias takes the accumulator's mean off.
    pad: an int or the 4-tuple (h0, h1, w0, w1)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    s_in, M = 2.0 ** -4, 0.5
    cg = c // group
    kk = cg * k * k
    zx, zw = (zx, zw) if u8 else (0, 0)
    ph0, ph1, pw0, pw1 = pad if isinstance(pad, tuple) else (pad,) * 4
    x = g.input(n, c, h, w, s_in, zx)
    wd = rng.choice(np.array([-1, 1]), (oc, cg, k, k)) * (rng.random((oc, cg, k, k)) < min(1.0, 6.0 / kk))
    if u8 and ties._shift(zw, -1, 1):
        wd = np.abs(wd) * (1 if zw < 128 else -1)
    b = (np.round(t_mid / M) + rng.integers(-2, 3, oc)).astype(np.int32)
    s_w = M * s_out / s_in
    if u8:
        xin = (zx + ties._shift(zx, -2, 2) + rng.integers(-2, 3, (n, c, h, w))).astype(np.uint8)
        if ties._shift(zx, -2, 2) or ties._shift(zw, -1, 1):
            L = dict(group=group, stride_h=stride, stride_w=stride, dilation_h=1, dilation_w=1, pad_h0=ph0, pad_h1=ph1, pad_w0=pw0,
                     pad_w1=pw1)
            b = (b - np.rint(ties.conv_acc(xin, zw + wd, L, zx, zw).mean(axis=(0, 2, 3)))).astype(np.int32)
        y = g.conv(x, (zw + wd).astype(np.uint8), b, [s_w], s_out, zo, stride=stride, pad=pad, group=group,
                   activation=activation, recipe=recipe, weight_zero=zw)
    else:
        y = g.conv(x, wd.astype(np.int8), b, np.full(oc, s_w, np.float32), s_out, stride=stride, pad=pad, group=group,
                   activation=activation, recipe=recipe)
        xin = rng.integers(-2, 3, (n, c, h, w)).astype(np.int8)
        if min_byte:
            xin[rng.random(xin.shape) < ties.MIN_BYTE_FRAC] = -128
    g.mark_output(y)
    cs = ties.Case(("uint8" if u8 else "int8") + f"_act{activation}_r{recipe}_so{s_out}_n{n}c{c}_{h}x{w}_oc{oc}_k{k}", g, [xin],
                   min_tie_frac=0.05)
    cs.mode = ties.planned_mode(g, g.layers[0])
    return cs


def concat_n(rng, u8, chans, shape=(2, 5, 7), zps=None, zo=110, ratios=None, min_byte=False):
    """Concat of len(chans) inputs with s_in / s_out = 1/2, 1/4, 1/2, ... (t = q/2, q/4): inputs whose channel count and offset
    are multiples of 16 take the byte table, the others the bytewise path (engine.cu fill_concat_steps).  zps: the inputs' uint8
    zero points (default 120, 125, ...); ratios: s_in / s_out per input (1: an input whose quantisation may equal the output's,
    which the table path copies)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    n, h, w = shape
    ins, xs = [], []
    for i, c in enumerate(chans):
        zp = ((120 + 5 * i) if zps is None else zps[i]) if u8 else 0
        s = 2.0 ** -(5 + i % 2) if ratios is None else 2.0 ** -4 * ratios[i]
        ins.append(g.input(n, c, h, w, s, zp))
        xs.append(ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zp, min_byte=min_byte))
    g.mark_output(g.concat(ins, 2.0 ** -4, zo if u8 else 0))
    return ties.Case(("uint8" if u8 else "int8") + "_concat_" + "_".join(map(str, chans)), g, xs, min_tie_frac=0.10)


def relu_maxpool(rng, u8, c, slope_exp=None, shape=(2, 9, 11), zi=128, zo=110, min_byte=False):
    """(Leaky) ReLU, then a 3x3 / 2 max pooling keeping the ReLU's quantisation: the pooling folds the ReLU in as a byte table
    (engine.cu fuse_nodes) when the ReLU's output is read by the pooling alone."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi, zo = (zi, zo) if u8 else (0, 0)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -5, zi)
    y = g.relu(x, 2.0 ** -4, zo, negative_slope=0.0 if slope_exp is None else 2.0 ** -slope_exp)
    g.mark_output(g.pool(y, abi.POOL_MAX, 3, 2, 1))
    xs = [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zi, min_byte=min_byte)]
    return ties.Case(("uint8" if u8 else "int8") + f"_relu_maxpool_c{c}", g, xs, min_tie_frac=0.20)


def eltwise_relu(rng, u8, c, shape=(2, 9, 11), z0=120, z1=130, zo=110, elt=abi.ELT_SUM, min_byte=False):
    """Eltwise SUM (or PROD), then a ReLU with the eltwise's own quantisation: folded into the eltwise kernel (engine.cu
    fuse_nodes)."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    z0, z1, zo = (z0, z1, zo) if u8 else (0, 0, 0)
    n, h, w = shape
    s0, s1, so, r = (2.0 ** -4, 2.0 ** -5, 2.0 ** -4, 60) if elt == abi.ELT_SUM else (2.0 ** -3, 2.0 ** -3, 2.0 ** -2, 40)
    a = g.input(n, c, h, w, s0, z0)
    b = g.input(n, c, h, w, s1, z1)
    s = g.eltwise(a, b, so, zo, elt_type=elt)
    g.mark_output(g.relu(s))
    xs = [ties._in(rng, u8, (n, c, h, w), -r, r, zp=z0, min_byte=min_byte), ties._in(rng, u8, (n, c, h, w), -r, r, zp=z1,
                                                                                     min_byte=min_byte)]
    return ties.Case(("uint8" if u8 else "int8") + f"_eltwise_relu_c{c}", g, xs, min_tie_frac=0.05)


def unary(rng, u8, op, c, shape=(2, 9, 11), zi=128, zo=0, min_byte=False):
    """Sigmoid or hardswish (uint8 only, as in the reference) over the whole byte range of its input: a byte table built at
    prerun (engine.cu), compared with the oracle."""
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi, zo = (zi, zo) if u8 else (0, 0)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -4, zi)
    g.mark_output(g.sigmoid(x, 2.0 ** -8 if u8 else 2.0 ** -7, zo) if op == "sigmoid" else g.hardswish(x, 2.0 ** -4, zo))
    xs = [ties._in(rng, u8, (n, c, h, w), -127, 127, zp=zi, min_byte=min_byte)]
    return ties.Case(("uint8" if u8 else "int8") + f"_{op}_c{c}", g, xs)


def silu(rng, c, shape=(2, 9, 11)):
    """x * sigmoid(x) (int8 YOLOv5s' SiLU): the pair becomes one byte table (engine.cu fuse_nodes)."""
    g = GraphDef(abi.DT_INT8)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -4)
    s = g.sigmoid(x, 2.0 ** -7)
    g.mark_output(g.eltwise(x, s, 2.0 ** -4, elt_type=abi.ELT_PROD))
    return ties.Case(f"int8_silu_c{c}", g, [ties._in(rng, False, (n, c, h, w), -127, 127)])


def relu_same(rng, c, shape=(2, 9, 11)):
    """int8 ReLU keeping its input's quantisation (max(byte, 0): engine.cu's same-scale kernel) over inputs with -128."""
    g = GraphDef(abi.DT_INT8)
    n, h, w = shape
    x = g.input(n, c, h, w, 2.0 ** -4)
    g.mark_output(g.relu(x))
    return ties.Case(f"int8_relu_same_c{c}", g, [ties._in(rng, False, (n, c, h, w), -127, 127, min_byte=True)])


def softmax(rng, u8, c, h=1, w=1, n=3, zi=128, min_byte=False):
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    zi = zi if u8 else 0
    x = g.input(n, c, h, w, 2.0 ** -4, zi)
    g.mark_output(g.softmax(x, 2.0 ** -7 if not u8 else 2.0 ** -8, 0))
    return ties.Case(("uint8" if u8 else "int8") + f"_softmax_c{c}_{h}x{w}", g,
                     [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zi, min_byte=min_byte)])


def upsample(rng, u8, c, scale, shape=(2, 5, 6), zi=128, min_byte=False):
    g = GraphDef(abi.DT_UINT8 if u8 else abi.DT_INT8)
    n, h, w = shape
    zi = zi if u8 else 0
    x = g.input(n, c, h, w, 2.0 ** -4, zi)
    g.mark_output(g.upsample(x, scale))
    return ties.Case(("uint8" if u8 else "int8") + f"_upsample{scale}_c{c}", g,
                     [ties._in(rng, u8, (n, c, h, w), -100, 100, zp=zi, min_byte=min_byte)])


G_, I_, D_, DD = "gemm_i8_tcgen05", "conv_igemm_i8_tcgen05", "conv_dw3x3_tma_dp4a", "conv_dw_direct"
LOW_M = (2, 2, 3, 4, 5)  # M_c >= 2^-2: the fast-path proof holds up to K ~ 1000
REF = abi.RECIPE_REF  # conv_recipe's for grouped convs, batched int8 and every uint8 depthwise

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
_add("dw3x3s1_i8_c144", _i8(2, 144, 13, 14, 144, k=3, pad=1, group=144, mode=1, recipe=REF), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s2_i8_c48", _i8(2, 48, 13, 14, 48, k=3, stride=2, pad=1, group=48, mode=0, recipe=REF), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s1_i8_c40", _i8(2, 40, 9, 10, 40, k=3, pad=1, group=40, mode=2, recipe=REF), D_, dict(valid=True, cp_mod32=16))
_add("dw3x3s1_i8_c64", _i8(2, 64, 9, 10, 64, k=3, pad=1, group=64, mode=1, recipe=REF), D_, dict(valid=True, cp_mod32=0))
_add("dw3x3s1_u8_c144", _u8(1, 144, 9, 10, 144, k=3, pad=1, group=144, recipe=REF), DD, dict(valid=False, cp_mod32=16))
# the row limit: 16 pixel groups (ow 128 at stride 1, 64 at stride 2); one more pixel takes the generic kernel
_add("dw3x3s1_i8_ow128", _i8(1, 48, 4, 128, 48, k=3, pad=1, group=48, mode=1), D_, dict(valid=True, gpr=16, stride=1))
_add("dw3x3s1_i8_ow129", _i8(1, 48, 4, 129, 48, k=3, pad=1, group=48, mode=1), DD, dict(valid=False, gpr=17, stride=1))
_add("dw3x3s2_i8_ow64", _i8(1, 48, 6, 128, 48, k=3, stride=2, pad=1, group=48, mode=1), D_, dict(valid=True, gpr=16, stride=2))
_add("dw3x3s2_i8_ow65", _i8(1, 48, 6, 129, 48, k=3, stride=2, pad=1, group=48, mode=1), DD, dict(valid=False, gpr=17, stride=2))
# fewer output rows than rows_per_cta
_add("dw3x3s1_i8_oh3_capped", _i8(2, 32, 3, 8, 32, k=3, pad=1, group=32, mode=1, recipe=REF), D_,
     dict(valid=True, rows_capped=True, rows_per_cta=3))
_add("dw3x3s1_i8_oh1_capped", _i8(3, 32, 1, 20, 32, k=3, pad=1, group=32, mode=0, recipe=REF), D_,
     dict(valid=True, rows_capped=True, rows_per_cta=1))
_add("dw3x3s2_i8_oh2_capped", _i8(2, 48, 3, 30, 48, k=3, stride=2, pad=1, group=48, mode=1, recipe=REF), D_,
     dict(valid=True, rows_capped=True))
_add("dw3x3s1_i8_oh17_full", _i8(1, 32, 17, 30, 32, k=3, pad=1, group=32, mode=1), D_, dict(valid=True, rows_capped=False, rows_per_cta=4))

# ---- NCHW stems: the window kernel (W % 16 == 0, stride 1 / 2) and the gather kernel -----------------------------------------
WI, GA, ST, DR = "conv_window_tcgen05", "conv_gather_tcgen05", "conv_stem_nchw_dp4a", "conv_direct_dp4a"
CONV_KERNELS = (G_, I_, D_, DD, WI, GA, ST, DR)  # FC layers run the GEMM too, and are never abi_only
NO_TC = abi.PRERUN_NO_TENSORCORE


def _both(name, n, c, h, w, oc, k, stride, pad, kernel, edges, group=1, recipe=abi.RECIPE_HCL, **kw):
    """The int8 and the uint8 entry of one conv shape (pad: an int or the 4-tuple (h0, h1, w0, w1)); modes as ties' defaults."""
    if isinstance(pad, tuple):
        _add(name.format("i8"), lambda r: i8_conv_pad(r, n, c, h, w, oc, k, stride, pad), kernel, edges, **kw)
        _add(name.format("u8"), lambda r: u8_conv_pad(r, n, c, h, w, oc, k, stride, pad), kernel, edges, **kw)
    else:
        _add(name.format("i8"), _i8(n, c, h, w, oc, k=k, stride=stride, pad=pad, group=group, recipe=recipe), kernel, edges, **kw)
        _add(name.format("u8"), _u8(n, c, h, w, oc, k=k, stride=stride, pad=pad, group=group, recipe=recipe), kernel, edges, **kw)


# 7x7 over 1 and 2 channels: 2 and 4 k-steps of A in shared memory (of the 5 a 147-byte row could fill), B right after them
_both("win7x7s2_{}_c1_p3", 2, 1, 21, 32, 24, 7, 2, 3, WI, dict(layout=1, ks=2, xoff=13, tiles_w=1, tw_magic0=True, tiles_h=2, ow_mod16=0))
_both("win7x7s2_{}_c2_p2", 3, 2, 30, 32, 24, 7, 2, 2, WI, dict(layout=1, ks=4, xoff=14, ow_mod16=15, batch1=False))
_both("win7x7s1_{}_c3_p0", 1, 3, 14, 32, 40, 7, 1, 0, WI, dict(layout=1, ks=5, xoff=0, tiles_w=2, tiles_h=1, th_magic0=True,
                                                                          oh_mod8=0, batch1=True))
_both("win7x7s1_{}_c1_p1", 1, 1, 22, 48, 24, 7, 1, 1, WI, dict(layout=1, ks=2, xoff=15, tiles_w=3, th_magic0=False))
_both("win3x3s1_{}_c1_p1", 2, 1, 15, 32, 24, 3, 1, 1, WI, dict(layout=0, ks=1, xoff=15, oh_mod8=7, tw_magic0=False, window_valid=True))
_both("win3x3s2_{}_c2_p2", 3, 2, 16, 64, 24, 3, 2, 2, WI, dict(layout=0, ks=1, xoff=14, ow_mod16=1, tiles_w=3))
_both("win3x3s2_{}_c3_pad01", 2, 3, 16, 32, 24, 3, 2, (0, 1, 0, 1), WI, dict(layout=0, xoff=0, ow_mod16=0, oh_mod8=0))
_both("win3x3s1_{}_c3_p3", 1, 3, 9, 32, 24, 3, 1, 3, WI, dict(layout=0, xoff=13, tiles_h=2, oh_mod8=5))
# W % 16 != 0 (no tensor map) or stride 3: the gather kernel; the last tile of 128 pixels full, one pixel, 127 pixels
_both("gat7x7s2_{}_c1_p3", 2, 1, 21, 30, 24, 7, 2, 3, GA, dict(ks=2, window_valid=False))
_both("gat7x7s1_{}_c2_p3", 1, 2, 12, 20, 24, 7, 1, 3, GA, dict(ks=4, npix_mod128=112))
_both("gat7x7s2_{}_c3_p3", 2, 3, 16, 24, 40, 7, 2, 3, GA, dict(ks=5))
_both("gat3x3s1_{}_c1_n2_8x8", 2, 1, 8, 8, 24, 3, 1, 1, GA, dict(ks=1, ntiles=1, npix_mod128=0))
_both("gat3x3s1_{}_c2_3x43", 1, 2, 3, 43, 24, 3, 1, 1, GA, dict(ks=1, ntiles=2, npix_mod128=1))
_both("gat3x3s1_{}_c3_5x51", 1, 3, 5, 51, 24, 3, 1, 1, GA, dict(ks=1, ntiles=2, npix_mod128=127))
_both("gat3x3s3_{}_c3_w32", 2, 3, 14, 32, 24, 3, 3, 1, GA, dict(ks=1, window_valid=False))
# the planner around the stems: OCp 256 is the tensor-core kernels' (a 7x7 window at xoff 13 no longer fits in shared memory),
# 272 the stem kernel's; 4 channels, a 5x5 kernel or a dilation take the stem kernel too (OCT 32 when OCp % 32 == 0, else 16)
_both("win7x7s2_{}_c3_oc256_p0", 1, 3, 16, 32, 256, 7, 2, 0, WI, dict(layout=1, ks=5, smem_bytes=203904))
_both("gat7x7s2_{}_c3_oc256_p3", 1, 3, 16, 32, 256, 7, 2, 3, GA, dict(ks=5, window_valid=False))
_both("win3x3s1_{}_c3_oc256", 1, 3, 8, 32, 256, 3, 1, 1, WI, dict(layout=0))
_both("stem3x3s1_{}_c3_oc272", 1, 3, 8, 32, 272, 3, 1, 1, ST, dict(oct=16))
_both("stem3x3s2_{}_c4", 2, 4, 11, 14, 32, 3, 2, 1, ST, dict(oct=32))
_both("stem5x5s2_{}_c3_oc48", 2, 3, 13, 15, 48, 5, 2, 2, ST, dict(oct=16))
_add("stem3x3d2_i8_c3", lambda r: i8_conv_pad(r, 2, 3, 12, 16, 24, 3, 1, 2, dilation=2), ST, dict(oct=32))
_add("stem3x3d2_u8_c3", lambda r: u8_conv_pad(r, 2, 3, 12, 16, 24, 3, 1, 2, dilation=2), ST, dict(oct=32))
_both("stem3x3s1_{}_c3_notc", 2, 3, 9, 16, 24, 3, 1, 1, ST, dict(oct=32), flags=NO_TC)

# ---- NHWC 16- and 32-byte pixels: the window kernel, the gather kernel past its limits, the implicit GEMM past window32's --------
_both("win3x3s1_{}_c16", 3, 16, 10, 20, 40, 3, 1, 1, WI, dict(layout=2, ks=5, tiles_w=2, tiles_h=2, batch1=False))
_both("win3x3s2_{}_c16_ocp224", 1, 16, 10, 12, 224, 3, 2, 1, WI, dict(layout=2, ks=5))
_both("gat3x3s2_{}_c16_ocp240", 1, 16, 10, 12, 240, 3, 2, 1, GA, dict(ks=5, window_valid=False))
_both("gat3x3s3_{}_c16", 2, 16, 11, 13, 40, 3, 3, 1, GA, dict(ks=5, window_valid=False))
_both("win3x3s1_{}_c32_ocp176", 1, 32, 8, 18, 176, 3, 1, 1, WI, dict(layout=3, ks=9))
_both("igemm3x3s1_{}_c32_ocp192", 1, 32, 8, 18, 192, 3, 1, 1, I_, dict(taps=9, block_k=32))
_both("win3x3s2_{}_c32_ocp144", 1, 32, 9, 20, 144, 3, 2, 1, WI, dict(layout=3, ks=9))
_both("igemm3x3s2_{}_c32_ocp160", 1, 32, 9, 20, 160, 3, 2, 1, I_, dict(taps=9))
# uint8 pad lanes (c >= C) inside a 16- / 32-byte pixel: the zero-point fill of border taps must leave them 0
_add("win3x3s1_u8_c8", _u8(3, 8, 9, 18, 40, k=3, pad=1), WI, dict(layout=2))
_add("gat3x3s3_u8_c12", _u8(2, 12, 10, 13, 40, k=3, stride=3, pad=1), GA, dict(ks=5))
_add("win3x3s2_u8_c24", _u8(3, 24, 9, 20, 40, k=3, stride=2, pad=1), WI, dict(layout=3, ks=9))

# ---- CUDA-core kernels: grouped direct conv (OCT 8 / 4), generic depthwise, the int8 depthwise 3x3 without a TMA plan -------
_both("direct3x3_{}_g4_og8", 2, 32, 7, 9, 32, 3, 1, 1, DR, dict(oct=8), group=4, recipe=REF)
_both("direct3x3_{}_g4_og12", 2, 32, 7, 9, 48, 3, 2, 1, DR, dict(oct=4), group=4, recipe=REF)
_add("dw5x5s1_i8_c32", _i8(2, 32, 9, 11, 32, k=5, pad=2, group=32, recipe=REF), DD, dict(valid=False, dw_kernel="generic"))
_add("dw3x3s2_u8_c32", _u8(2, 32, 9, 11, 32, k=3, stride=2, pad=1, group=32, recipe=REF), DD, dict(valid=False, dw_kernel="generic"))
_add("dw3x3s1_i8_c32_notc", _i8(2, 32, 7, 13, 32, k=3, pad=1, group=32, recipe=REF), DD, dict(dw_kernel="dw3x3_i8", dw_ow_tail=5),
     flags=NO_TC)
_add("dw3x3s2_i8_c48_notc", _i8(2, 48, 9, 13, 48, k=3, stride=2, pad=1, group=48, mode=0, recipe=REF), DD,
     dict(dw_kernel="dw3x3_i8", dw_ow_tail=3), flags=NO_TC)
_add("dw3x3s1_i8_c32_w16_notc", _i8(1, 32, 5, 16, 32, k=3, pad=1, group=32), DD, dict(dw_kernel="dw3x3_i8", dw_ow_tail=0), flags=NO_TC)

# ---- activation clamps in the epilogues: ReLU and ReLU6 (HCL), [-1, 1] and ReLU6 (REF) ------------------------------------------
# s_out = 4 puts ReLU6's bound at t = 1.5, s_out = 2 REF's [-1, 1] at t = +-0.5: half-integer bounds, which the reference's
# round() takes away from zero; [-1, 1] is the only clamp whose lower integer bound is neither 0 nor -127 (int8: q_byte_add 0xff)
ACTS = {"hcl0": (0, abi.RECIPE_HCL, 2.0 ** -2), "hcl6": (6, abi.RECIPE_HCL, 4.0), "ref1": (1, abi.RECIPE_REF, 2.0),
        "ref6": (6, abi.RECIPE_REF, 4.0)}
_ACT_SHAPES = {  # kernel, (n, c, h, w, oc, k, stride, pad, group), dtypes
    "win3x3": (WI, (2, 3, 9, 32, 24, 3, 1, 1, 1), ("i8", "u8")),
    "gat3x3": (GA, (2, 3, 9, 30, 24, 3, 1, 1, 1), ("i8", "u8")),
    "stem3x3": (ST, (2, 4, 9, 11, 24, 3, 1, 1, 1), ("i8", "u8")),
    "gemm1x1": (G_, (2, 64, 9, 7, 40, 1, 1, 0, 1), ("i8", "u8")),
    "dw3x3": (D_, (2, 32, 9, 10, 32, 3, 1, 1, 32), ("i8",)),
}
# Every recipe on every kernel, so also the ones Tengine never picks for the shape (conv_recipe: HCL for group 1, REF for the
# batched depthwise): those are abi_only.
for sh, (kern, (n, c, h, w, oc, k, st, pd, gp), dts) in _ACT_SHAPES.items():
    for a, (act, rec, so) in ACTS.items():
        for d in dts:
            edges = dict(act=a, bound_half=a != "hcl0", bound_beyond_sat=False)
            if kern == D_:
                edges["valid"] = True
            _add(f"{sh}_{d}_{a}", lambda r, d=d, act=act, rec=rec, so=so, n=n, c=c, h=h, w=w, oc=oc, k=k, st=st, pd=pd, gp=gp:
                 act_conv(r, d == "u8", n, c, h, w, oc, act, rec, so, k=k, stride=st, pad=pd, group=gp, t_mid=0.75), kern, edges,
                 abi_only=(rec == REF) == (gp == 1))
# bounds beyond the byte range: ReLU6 at t = 192 > 127 (int8); uint8 output zero points 254 (ReLU6's 2 + 254 > 255) and 0
# ([-1, 1]'s -1 + 0 < 0)
_add("win3x3_i8_hcl6_sat", lambda r: act_conv(r, False, 2, 3, 9, 32, 24, 6, abi.RECIPE_HCL, 2.0 ** -5, t_mid=126.5), WI,
     dict(act="hcl6", bound_half=False, bound_beyond_sat=True))
_add("win3x3_u8_hcl6_zo254", lambda r: act_conv(r, True, 2, 3, 9, 32, 24, 6, abi.RECIPE_HCL, 4.0, zo=254, t_mid=0.75), WI,
     dict(act="hcl6", bound_half=True, bound_beyond_sat=True))
_add("gat3x3_u8_ref1_zo0", lambda r: act_conv(r, True, 2, 3, 9, 30, 24, 1, abi.RECIPE_REF, 2.0, zo=0), GA,
     dict(act="ref1", bound_half=True, bound_beyond_sat=True), abi_only=True)
_add("stem3x3_u8_ref6_zo254", lambda r: act_conv(r, True, 2, 4, 9, 11, 24, 6, abi.RECIPE_REF, 4.0, zo=254, t_mid=0.75), ST,
     dict(act="ref6", bound_beyond_sat=True), abi_only=True)
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

# ---- the ends of the byte range: uint8 zero points 0, 1, 128 and 255 -----------------------------------------------------------
# The uint8 GEMM's operand regime follows the weight zero point (gemm_tcgen05.cu plan_begin): zw 0 -> B holds the plain weights,
# unsigned (the u8.u8 MMA), no cplane term; zw 128 -> cplane 0, no row-sum warps; else B holds w - 128 and cplane = 128 - zw adds
# cplane * sum(x) from the row sums (+127 at zw 1, -127 at zw 255).  Each regime through the 1x1 GEMM, an FC over C % 16 != 0,
# the implicit GEMM with padding (border table), several N tiles, streamed B (b_res 0), MODE 0 and MODE 2.  The MODE 0 entries
# keep x about a mid zero point (one-sided x and w would put the bias past the fast path's bound); the MODE 2 ones move x to an
# end of the byte range too.
U8_REGIMES = {"zw0": (0, "unsigned_b", 255), "zw128": (128, "no_cplane", 0), "zw1": (1, "cplane_max", 255),
              "zw255": (255, "cplane_min", 0)}
for rg, (zw, ops, zx_end) in U8_REGIMES.items():
    def _r(edges, **kw):
        return dict(edges, u8_operands=ops, b_signed=int(zw != 0), cplane=0 if zw in (0, 128) else 128 - zw, **kw)
    _add(f"gemm1x1_u8_{rg}", _u8(2, 64, 9, 7, 40, zw=zw), G_, _r(dict(b_res=1, n_tiles=1)))
    _add(f"gemm1x1_u8_{rg}_zx{zx_end}_m2", _u8(2, 64, 9, 7, 40, zw=zw, zx=zx_end, mode=2), G_, _r(dict(zx=zx_end)))
    _add(f"gemm1x1_u8_{rg}_ocp400", _u8(2, 64, 9, 7, 400, zw=zw), G_, _r(dict(n_tiles=4, n_uneven=True)))
    _add(f"fc_u8_c24_3x3_{rg}", lambda r, zw=zw: ties.uint8_conv(r, 3, 24, 3, 3, 50, fc=True, zw=zw), G_, _r(dict(k_blocks=3)))
    _add(f"fc_u8_k4608_{rg}_m2", lambda r, zw=zw: ties.uint8_conv(r, 2, 512, 3, 3, 64, fc=True, mode=2, zw=zw), G_,
         _r(dict(b_res=0, k_blocks=36)))
    _add(f"igemm3x3_u8_{rg}_m2", _u8(2, 64, 9, 10, 40, k=3, pad=1, mode=2, zw=zw), I_, _r(dict(border=1, taps=9)))
    _add(f"igemm7x7_u8_{rg}_m2", _u8(1, 64, 13, 12, 40, k=7, pad=3, mode=2, zw=zw), I_, _r(dict(border=1, taps=49)))
# every (block_n, mt) of gemm_mma_dispatch on the unsigned-B path: one N tile of OCp = block_n channels; mt 2 over 3 m-tiles, mt 4
# (block_n <= 32) over 5
MMA_PAIRS = ((16, 1), (16, 2), (16, 4), (32, 1), (32, 2), (32, 4), (48, 1), (48, 2), (64, 1), (64, 2), (80, 1), (96, 1), (112, 1),
             (128, 1))
for bn, mt in MMA_PAIRS:
    shp = {1: (1, 10, 12), 2: (1, 15, 20), 4: (2, 15, 20)}[mt if bn < 80 else 2]
    _add(f"gemm1x1_u8_zw0_bn{bn}_mt{mt}", _u8(shp[0], 32, shp[1], shp[2], bn, zw=0), G_,
         dict(mma_uu=(bn, mt), block_n=bn, mt=mt, b_signed=0, cplane=0))
# the largest accumulators: |x - zx| = |w - zw| in [235, 255] at K = 4608 (3x3x512, padded) and 25088 (VGG fc6), both operand
# regimes with a non-zero correction term away from zx = 0: unsigned B (zx 255, zw 0) and cplane -127 (zx 0, zw 255)
for zx, zw in ((255, 0), (0, 255)):
    _add(f"igemm3x3_u8_far_z{zx}_{zw}", lambda r, zx=zx, zw=zw: u8_far(r, 1, 512, 10, 10, 64, k=3, pad=1, zx=zx, zw=zw, s_out=16.0),
         I_, dict(k_blocks=36, border=1, zx=zx, b_signed=int(zw != 0)), ref="oracle", ties=False)
    _add(f"fc_u8_far_z{zx}_{zw}", lambda r, zx=zx, zw=zw: u8_far(r, 2, 512, 7, 7, 64, fc=True, zx=zx, zw=zw, s_out=32.0),
         G_, dict(k_blocks=196, b_res=0, zx=zx, b_signed=int(zw != 0)), ref="oracle", ties=False)
# zx = 255: the window and gather kernels fill out-of-image taps with 0xFF, the implicit GEMM's border table holds its largest
# corrections; zx = 0 likewise
for zx in (0, 255):
    _add(f"win3x3s1_u8_c3_zx{zx}", _u8(2, 3, 15, 32, 24, k=3, pad=1, zx=zx), WI, dict(layout=0, zx=zx))
    _add(f"win7x7s2_u8_c3_zx{zx}", _u8(2, 3, 21, 32, 24, k=7, stride=2, pad=3, zx=zx), WI, dict(layout=1, zx=zx))
    _add(f"win3x3s1_u8_c16_zx{zx}", _u8(3, 16, 10, 20, 40, k=3, pad=1, zx=zx), WI, dict(layout=2, zx=zx))
    _add(f"win3x3s2_u8_c24_zx{zx}", _u8(3, 24, 9, 20, 40, k=3, stride=2, pad=1, zx=zx), WI, dict(layout=3, zx=zx))
    _add(f"gat3x3s1_u8_c3_zx{zx}", _u8(2, 3, 14, 30, 24, k=3, pad=1, zx=zx), GA, dict(ks=1, zx=zx, window_valid=False))
    _add(f"gat7x7s2_u8_c3_zx{zx}", _u8(2, 3, 16, 24, 40, k=7, stride=2, pad=3, zx=zx), GA, dict(ks=5, zx=zx, window_valid=False))
    _add(f"igemm3x3_u8_zx{zx}_m2", _u8(2, 64, 9, 10, 40, k=3, pad=1, mode=2, zx=zx), I_, dict(border=1, zx=zx))
    _add(f"direct3x3_u8_c32_notc_zx{zx}", _u8(2, 32, 7, 9, 32, k=3, pad=1, zx=zx), DR, dict(oct=8, zx=zx), flags=NO_TC)
    _add(f"dw3x3s1_u8_c32_zx{zx}", _u8(2, 32, 9, 11, 32, k=3, pad=1, group=32, zx=zx, recipe=REF), DD,
         dict(dw_kernel="generic", zx=zx))
    _add(f"dw3x3s2_u8_c32_zx{zx}", _u8(2, 32, 9, 11, 32, k=3, stride=2, pad=1, group=32, zx=zx, recipe=REF), DD,
         dict(dw_kernel="generic", zx=zx))
    _add(f"direct3x3d2_u8_c32_zx{zx}", lambda r, zx=zx: u8_conv_pad(r, 2, 32, 12, 16, 24, 3, 1, 2, dilation=2, zx=zx), DR,
         dict(oct=8, zx=zx))
# output zero points 0 and 255 under every activation: make_epi saturates the clamp's bounds before it builds the fast
# epilogue's constants.  t about t_mid; at zo 255 the ReLU-type clamps leave only t <= 0.5, so every byte is 255 (no live ties)
_ZO_ACTS = dict(ACTS, none=(-1, abi.RECIPE_HCL, 1.0))
_ZO_SHAPES = {"gemm1x1": (G_, (2, 64, 9, 7, 40, 1, 1, 0, 1)), "win3x3": (WI, (2, 3, 9, 32, 24, 3, 1, 1, 1)),
              "direct3x3": (DR, (2, 32, 7, 9, 32, 3, 1, 1, 4))}
for sh, (kern, (n, c, h, w, oc, k, st, pd, gp)) in _ZO_SHAPES.items():
    for a, (act, rec, so) in _ZO_ACTS.items():
        if a == "none":
            rec = abi.RECIPE_HCL if gp == 1 else REF  # no clamp: the recipe Tengine gives the shape (conv_recipe)
        for zo in (0, 255):
            t_mid = {"none": 20.0 if zo == 0 else -20.0, "ref1": 0.0}.get(a, 0.75)
            dense = zo == 0 or a in ("none", "ref1")
            _add(f"{sh}_u8_{a}_zo{zo}", lambda r, act=act, rec=rec, so=so, zo=zo, t_mid=t_mid, n=n, c=c, h=h, w=w, oc=oc, k=k, st=st,
                 pd=pd, gp=gp: act_conv(r, True, n, c, h, w, oc, act, rec, so, k=k, stride=st, pad=pd, group=gp, zo=zo, t_mid=t_mid),
                 kern, dict(act=a, zo=zo), ties=dense, notes={} if dense else dict(constant_output=True), abi_only=(rec == REF) == (gp == 1))
# The REF clamps where Tengine itself runs conv_ref (conv_recipe): grouped direct convs (OCT 8 and 4), the uint8 generic
# depthwise, and int8 depthwise convs at batch 1 that conv_dw_hcl_x86 turns down (one-sided padding on one axis, a 5x5 kernel).
# Tie-dense at the half-integer bounds, so that the reference itself says where a clamped value rounds.
_REF_SHAPES = {  # name ({} = dtype), kernel, (n, c, h, w, oc, k, stride, pad, group), dtypes, edges
    "direct3x3_{}_g4_og8": (DR, (2, 32, 7, 9, 32, 3, 1, 1, 4), ("i8", "u8"), dict(oct=8)),
    "direct3x3_{}_g4_og12": (DR, (2, 32, 7, 9, 48, 3, 2, 1, 4), ("i8", "u8"), dict(oct=4)),
    "dw3x3s1_{}_c32": (DD, (2, 32, 9, 11, 32, 3, 1, 1, 32), ("u8",), dict(dw_kernel="generic")),
    "dw3x3s2_{}_c32": (DD, (2, 32, 9, 11, 32, 3, 2, 1, 32), ("u8",), dict(dw_kernel="generic")),
    "dw3x3s1_{}_n1_pad0111": (D_, (1, 32, 9, 11, 32, 3, 1, (0, 1, 1, 1), 32), ("i8",), dict(valid=True)),
    "dw5x5s1_{}_n1": (DD, (1, 32, 9, 11, 32, 5, 1, 2, 32), ("i8",), dict(dw_kernel="generic")),
}
for sh, (kern, (n, c, h, w, oc, k, st, pd, gp), dts, edges) in _REF_SHAPES.items():
    for a in ("ref1", "ref6"):
        act, _, so = ACTS[a]
        for d in dts:
            _add(sh.format(d) + "_" + a, lambda r, d=d, act=act, so=so, n=n, c=c, h=h, w=w, oc=oc, k=k, st=st, pd=pd, gp=gp:
                 act_conv(r, d == "u8", n, c, h, w, oc, act, REF, so, k=k, stride=st, pad=pd, group=gp, t_mid=0.75), kern,
                 dict(edges, act=a, bound_half=True, bound_beyond_sat=False))
# and [-1, 1] at uint8 output zero points 0 and 255 (t about 0: both bounds live)
for sh in ("direct3x3_{}_g4_og12", "dw3x3s2_{}_c32"):
    kern, (n, c, h, w, oc, k, st, pd, gp), _, edges = _REF_SHAPES[sh]
    for zo in (0, 255):
        _add(sh.format("u8") + f"_ref1_zo{zo}", lambda r, zo=zo, n=n, c=c, h=h, w=w, oc=oc, k=k, st=st, pd=pd, gp=gp:
             act_conv(r, True, n, c, h, w, oc, 1, REF, 2.0, k=k, stride=st, pad=pd, group=gp, zo=zo, t_mid=0.0), kern,
             dict(edges, act="ref1", zo=zo, bound_beyond_sat=True))

# glue ops at the ends of the byte range
_PW, _CR, _LUT = "pointwise", "concat_requant", "byte_lut"
# uint8 pooling has no lower clamp: below 0 (zo < zi) the result wraps
_add("avgpool2x2s2_u8_wrap", lambda r: ties.pool(r, True, abi.POOL_AVG, 2, 2, zi=255, zo=0), _P, dict(pool_wraps=True, zx=255, zo=0))
_add("maxpool3x3s2_u8_wrap", lambda r: ties.pool(r, True, abi.POOL_MAX, 3, 2, pad=1, scale_ratio=2, zi=255, zo=0, shape=(2, 20, 9, 10)),
     _P, dict(pool_wraps=True, zx=255, zo=0))
_add("avgpool2x2s2_u8_zi0", lambda r: ties.pool(r, True, abi.POOL_AVG, 2, 2, zi=0, zo=60), _P, dict(pool_wraps=False, zx=0))
_add("maxpool2x3s1_u8_zi255", lambda r: ties.pool(r, True, abi.POOL_MAX, (2, 3), 1, scale_ratio=2, zi=255, zo=255), _P,
     dict(pool_wraps=False, zx=255))
# ReLU and leaky ReLU with zi 255 (every input at or below the zero point) or zo 0
_add("relu_u8_zi255", lambda r: ties.relu(r, True, zi=255, zo=110), _PW, dict(zx=255), ties=False)
_add("relu_u8_zo0", lambda r: ties.relu(r, True, zi=128, zo=0), _PW, dict(zo=0))
_add("leaky_relu_u8_zi255", lambda r: ties.relu(r, True, slope_exp=1, zi=255, zo=110), _PW, dict(zx=255))
_add("leaky_relu_u8_zo0", lambda r: ties.relu(r, True, slope_exp=2, zi=128, zo=0), _PW, dict(zo=0))
# eltwise sum and product with zero points 0 and 255, and with the folded ReLU
_add("eltwise_sum_u8_z0_255_zo0", lambda r: ties.eltwise(r, True, abi.ELT_SUM, z0=0, z1=255, zo=0), _PW, dict(zx=0, zo=0))
_add("eltwise_sum_u8_z255_0_zo255", lambda r: ties.eltwise(r, True, abi.ELT_SUM, z0=255, z1=0, zo=255), _PW, dict(zx=255, zo=255))
_add("eltwise_prod_u8_z0_255_zo255", lambda r: ties.eltwise(r, True, abi.ELT_PROD, z0=0, z1=255, zo=255), _PW, dict(zx=0, zo=255))
_add("eltwise_prod_u8_z255_255_zo0", lambda r: ties.eltwise(r, True, abi.ELT_PROD, z0=255, z1=255, zo=0), _PW, dict(zx=255, zo=0))
_add("eltwise_relu_u8_z0_255_zo0", lambda r: eltwise_relu(r, True, 32, z0=0, z1=255, zo=0), _F, dict(zx=0, zo=0), layer=1, fused=True,
     tie_layer=0)
_add("eltwise_prod_relu_u8_z255_255_zo0", lambda r: eltwise_relu(r, True, 32, z0=255, z1=255, zo=0, elt=abi.ELT_PROD), _F,
     dict(zx=0, zo=0), layer=1, fused=True, tie_layer=0)
# concat through the byte table and the bytewise kernel, zero points 0 and 255 in and out; an input with the output's quantisation
# takes the table path without a table (a copy)
for z in (0, 255):
    _add(f"concat4_u8_z{z}", lambda r, z=z: concat_n(r, True, (16, 8, 24, 16), zps=(z,) * 4, zo=z), _CR, dict(mixed=True, zx=z, zo=z))
    _add(f"concat3_aligned_u8_z{z}", lambda r, z=z: concat_n(r, True, (16, 32, 16), zps=(z,) * 3, zo=z), _CR, dict(mixed=False, zx=z, zo=z))
_add("concat2_aligned_u8_copy_z255", lambda r: concat_n(r, True, (16, 32), zps=(255, 255), zo=255, ratios=(1, 0.5)), _CR,
     dict(mixed=False, zx=255, zo=255))
# the ReLU folded into max pooling as a table, at zo 255: a plain ReLU saturates every byte, a leaky one keeps its negative side
_add("relu_maxpool_u8_c32_zo255", lambda r: relu_maxpool(r, True, 32, zi=128, zo=255), _F, dict(zo=255), fused=True, tie_layer=0,
     ties=False)
_add("leaky_relu_maxpool_u8_c32_zi255_zo255", lambda r: relu_maxpool(r, True, 32, slope_exp=1, zi=255, zo=255), _F,
     dict(zx=255, zo=255), fused=True, tie_layer=0)
# byte tables and softmax over inputs at zi 255
_add("sigmoid_u8_c24_zi255", lambda r: unary(r, True, "sigmoid", 24, zi=255), _LUT, dict(zx=255), ref="oracle", ties=False)
_add("hardswish_u8_c24_zi255", lambda r: unary(r, True, "hardswish", 24, zi=255, zo=128), _LUT, dict(zx=255), ref="oracle",
     ties=False)
_add("softmax_c21_5x6_u8_zi255", lambda r: softmax(r, True, 21, 5, 6, zi=255), "softmax", dict(zx=255), ref="oracle", ties=False)

# ---- int8 -128 in a graph input: the reference clamps it to -127 in every op, its concat to +127 (concat_kernel_ref_int8.c:77-78) ----
_M = dict(in_min_byte=True)
# concat: an input with the output's quantisation (the table path's copy), the bytewise kernel at the same scale, and rescaled
_add("concat2_aligned_i8_copy", lambda r: concat_n(r, False, (16, 32), ratios=(1, 0.5)), _CR, dict(in_min_byte=False, mixed=False))
_add("concat2_aligned_i8_copy_min", lambda r: concat_n(r, False, (16, 32), ratios=(1, 0.5), min_byte=True), _CR, dict(_M, mixed=False))
_add("concat2_i8_bytewise_same_min", lambda r: concat_n(r, False, (8, 24), ratios=(1, 1), min_byte=True), _CR, dict(_M, mixed=False),
     ties=False)
_add("concat3_i8_min", lambda r: concat_n(r, False, (32, 40, 16), min_byte=True), _CR, dict(_M, mixed=True))
# pooling: max at the same scale (the byte path), max rescaled, average
_add("maxpool3x3s2_i8_same_min", lambda r: ties.pool(r, False, abi.POOL_MAX, 3, 2, pad=1, shape=(2, 32, 9, 10), min_byte=True), _P,
     dict(_M), ties=False)
_add("maxpool2x3s1_i8_min", lambda r: ties.pool(r, False, abi.POOL_MAX, (2, 3), 1, scale_ratio=2, min_byte=True), _P, dict(_M))
_add("avgpool2x2s2_i8_min", lambda r: ties.pool(r, False, abi.POOL_AVG, 2, 2, min_byte=True), _P, dict(_M))
# ReLU at the same scale, leaky ReLU, eltwise sum and product, sigmoid (int8 has no hardswish in the reference), softmax, upsample
_add("relu_same_i8_min", lambda r: relu_same(r, 32), _PW, dict(_M), ties=False)
_add("leaky_relu_i8_min", lambda r: ties.relu(r, False, slope_exp=2, min_byte=True), _PW, dict(_M))
_add("eltwise_sum_i8_min", lambda r: ties.eltwise(r, False, abi.ELT_SUM, min_byte=True), _PW, dict(_M))
_add("eltwise_prod_i8_min", lambda r: ties.eltwise(r, False, abi.ELT_PROD, min_byte=True), _PW, dict(_M))
_add("sigmoid_i8_c24_min", lambda r: unary(r, False, "sigmoid", 24, min_byte=True), _LUT, dict(_M), ref="oracle", ties=False)
_add("softmax_c21_5x6_i8_min", lambda r: softmax(r, False, 21, 5, 6, min_byte=True), "softmax", dict(_M), ref="oracle", ties=False)
_add("upsample2_c24_i8_min", lambda r: upsample(r, False, 24, 2, min_byte=True), "upsample_nearest", dict(_M), ref="oracle", ties=False)
# convolutions reading the graph input: the stem's window and gather kernels, the GEMM on its NHWC copy, the depthwise kernels
_add("win3x3s1_i8_c3_min", _i8(2, 3, 15, 32, 24, k=3, pad=1, min_byte=True), WI, dict(_M, layout=0))
_add("gat3x3s1_i8_c3_min", _i8(2, 3, 14, 30, 24, k=3, pad=1, min_byte=True), GA, dict(_M, window_valid=False))
_add("gemm1x1_i8_min", _i8(2, 64, 9, 7, 40, mode=1, min_byte=True), G_, dict(_M))
_add("dw3x3s1_i8_c32_min", _i8(2, 32, 9, 10, 32, k=3, pad=1, group=32, min_byte=True, recipe=REF), D_, dict(_M, valid=True))
_add("dw5x5s1_i8_c32_min", _i8(2, 32, 9, 11, 32, k=5, pad=2, group=32, min_byte=True, recipe=REF), DD, dict(_M, dw_kernel="generic"))

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
    # the window and the gather kernel
    "layout": {0, 1, 2, 3},
    "ks": {1, 2, 4, 5, 9},
    "xoff": {0, 13, 14, 15},
    "window_valid": {True, False},
    "tw_magic0": {True, False},
    "th_magic0": {True, False},
    "batch1": {True, False},
    "ow_mod16": {0, 1, 15},
    "oh_mod8": {0, 7},
    "npix_mod128": {0, 1, 127},
    # the CUDA-core kernels
    "oct": {4, 8, 16, 32},
    "dw_kernel": {"dw3x3_i8", "generic"},
    "dw_ow_tail": {0, 3, 5},
    # the epilogue's clamp
    "act": {"hcl0", "hcl6", "ref1", "ref6"},
    "bound_half": {True, False},
    "bound_beyond_sat": {True, False},
    # the ends of the byte range
    "u8_operands": {"unsigned_b", "no_cplane", "cplane_max", "cplane_min"},
    "mma_uu": set(MMA_PAIRS),
    "zx": {0, 255},
    "zo": {0, 255},
    "pool_wraps": {True, False},
    "in_min_byte": {True, False},
    # a conv entry whose recipe only a C-ABI caller can ask for (Entry.abi_only), and one with the recipe Tengine picks
    "abi_only": {True, False},
}

# Edges no graph can reach, and why (none so far).
UNREACHABLE = {}

# Entries on which the device's arithmetic (the oracle's uint8 mode 0: the exact integer sum) and the unmodified reference differ
# by more than 1 LSB: entry -> (layer, the largest difference in LSB, why).  The reference's fp32 simulation (oracle mode 1) equals
# the reference on every one of them.
REFERENCE_DIVERGENCES = {
    name: (0, 15, "K = 25088 and |x - zx| = |w - zw| >= 235: the reference sums the products in fp32, which rounds once the sum "
                  "passes 2^24 (|acc| ~ 1.5e9 here); the device keeps the exact integer sum")
    for name in ("fc_u8_far_z255_0", "fc_u8_far_z0_255")
}


def reference_entries():
    """The entries the unmodified reference can judge: every one but the abi_only convs."""
    return [n for n, e in ENTRIES.items() if not e.abi_only]


def gemm_entries():
    return [n for n, e in ENTRIES.items() if e.kernel in (G_, I_)]


def uint8_gemm_entries():
    return [n for n in gemm_entries() if "_u8_" in n or n.startswith("fc_u8")]


def negative_control_entries():
    """The uint8 GEMM entries whose output is not one constant byte (a saturated output cannot show a wrong accumulator), and
    whether the restated plan has a cplane term: without it (TB200_DEBUG_NO_CPLANE) exactly those with one must fail."""
    out = {}
    for n in uint8_gemm_entries():
        if ENTRIES[n].notes.get("constant_output"):
            continue
        case = build(n)
        out[n] = gemm_geometry_of(case, ENTRIES[n])["cplane"] != 0
    return out


def gemm_geometry_of(case, e):
    return geometry(case.g, case.g.layers[e.layer])


def window_entries():
    """The window and gather entries: the GPU test ties their printed plans to window_geometry / gather_geometry."""
    return [n for n, e in ENTRIES.items() if e.kernel in (WI, GA)]


def window_batch_entries():
    """Window entries of 3 or more images: run again on all images but the last (tb200_graph_set_batch), where every slice's
    tensor map is built from its own n."""
    return [n for n in window_entries() if ENTRIES[n].kernel == WI and build(n).g.tensors[0]["dims"][0] >= 3]
