"""Every requantising epilogue on the device against the exact reference of tests/ties.py, on tie-dense layers.

With power-of-two scales a large share of the outputs are exact ties, where the fast epilogues' round-half-to-even differs from
the reference's round-half-away: each case first shows that round half to even would change its bytes, then requires every
byte of every layer to equal the exact reference.  So a tie guard or rare path that is missing, writes the wrong byte or the
wrong address, fails here by construction -- not by chance on a few elements of a big network.

Each case reaches its kernel by its shape; test_every_compiled_instantiation_is_launched runs them all in a child process
(`python -m tests.test_gpu_requant_ties <case>...`) with TB200_DEBUG_LAUNCH, which the library reads once per process."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tengine_b200 import abi
from tests import ties

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, R = abi.RECIPE_HCL, abi.RECIPE_REF
FIXQ_CAP = 4096  # entries of the deferred rare-path queue per CTA (engine.cu)
MARK = "requant_ties case "


def _rng(name):
    return np.random.default_rng(sum(name.encode()) * 7919)


# name -> (builder, prerun flags).  Builders take an rng.
def _i8(*a, **k):
    return lambda r: ties.int8_conv(r, *a, **k)


def _u8(*a, **k):
    return lambda r: ties.uint8_conv(r, *a, **k)


CASES = {}


def _add(name, build, flags=0):
    CASES[name] = (build, flags)


# ---- persistent GEMM (gemm_i8_tcgen05_kernel<U8, MODE, CS, BORDER>) ----
# 1x1 (flat GEMM), ragged M (2*15*15 = 450 rows), 128-channel N tile (8 chunks: the planner picks CS 2), odd OC
for mode in (0, 1, 2):
    _add(f"gemm1x1_i8_m{mode}_cs2", _i8(2, 64, 15, 15, 125, mode=mode))
for mode in (0, 2):
    _add(f"gemm1x1_u8_m{mode}_cs2", _u8(2, 64, 15, 15, 125, mode=mode))
    # uint8 with padding: BORDER corrections (implicit GEMM, 3x3, out_mode 1; 64-channel N tile, 2 m-tiles a stage: CS 2)
    _add(f"igemm3x3_u8_border_m{mode}_cs2", _u8(2, 64, 17, 19, 61, k=3, pad=1, mode=mode))
# implicit GEMM output modes: 0 (several images per m-tile), 1 (ow <= 128), 2 (ow > 128, ragged last tile of each row)
for mode in (0, 1, 2):
    _add(f"igemm_i8_outmode0_m{mode}", _i8(5, 64, 7, 7, 48, k=3, pad=1, mode=mode))
    _add(f"igemm_i8_outmode1_m{mode}", _i8(2, 64, 21, 19, 40, k=3, pad=1, mode=mode))
    _add(f"igemm_i8_outmode2_m{mode}", _i8(1, 64, 4, 150, 40, k=3, pad=1, mode=mode, activation=0))
    _add(f"igemm_i8_1x1s2_m{mode}", _i8(2, 64, 19, 23, 24, k=1, stride=2, mode=mode, recipe=R, activation=6))
for mode in (0, 2):
    _add(f"igemm_u8_outmode0_m{mode}", _u8(5, 64, 7, 7, 48, k=3, pad=1, mode=mode))
    _add(f"igemm_u8_outmode2_m{mode}", _u8(1, 64, 4, 150, 40, k=3, pad=1, mode=mode, recipe=R))
    _add(f"igemm_u8_1x1s2_noborder_m{mode}", _u8(2, 64, 19, 23, 24, k=1, stride=2, mode=mode))
# several N tiles: weights resident (K = 64) and streamed (K = 1024)
_add("gemm_i8_ntiles2_resident", _i8(2, 64, 13, 11, 250, mode=1))
_add("gemm_i8_ntiles2_streamed", _i8(1, 1024, 9, 9, 250, mode=0, m_exps=(2, 2, 2, 3, 4, 5, 6, 7, 8)))  # (M = 2^-1 fails the proof at K = 1024)
_add("gemm_u8_ntiles2_streamed", _u8(1, 512, 9, 9, 250))
# ---- FC (persistent GEMM over one row per image) ----
for mode in (0, 2):
    _add(f"fc_i8_m{mode}", lambda r, m=mode: ties.int8_fc(r, 5, 512, 200, mode=m))
    _add(f"fc_u8_m{mode}", lambda r, m=mode: ties.uint8_conv(r, 5, 32, 2, 2, 200, fc=True, mode=m))
# ---- the other tensor-core families ----
# The window kernel takes NCHW stems whose width is a multiple of 16, and 3x3 convolutions whose window fits in shared memory
# (conv_window.cu window_smem_bytes: 41856 + 680 OCp bytes for 16 input channels at stride 2, at most 204800, so OC <= 224);
# the gather kernel takes the rest.
for mode in (0, 1, 2):
    for tag, w in (("window", 32), ("gather", 34)):
        _add(f"stem3x3_i8_{tag}_m{mode}", _i8(2, 3, 24, w, 40, k=3, stride=2, pad=1, mode=mode, activation=0))
    _add(f"stem3x3_i8_w30_m{mode}", _i8(2, 3, 22, 30, 40, k=3, stride=1, pad=1, mode=mode))
    for tag, w in (("window", 32), ("gather", 34)):
        _add(f"stem7x7_i8_{tag}_m{mode}", _i8(2, 3, 30, w, 24, k=7, stride=2, pad=3, mode=mode))
    for tag, s, oc in (("window", 1, 40), ("gather", 2, 240), ("window_s2", 2, 224)):
        _add(f"nhwc16_3x3_i8_{tag}_m{mode}", _i8(2, 16, 15, 17, oc, k=3, stride=s, pad=1, mode=mode, recipe=R))
    _add(f"nhwc32_3x3_i8_window_m{mode}", _i8(2, 32, 18, 18, 40, k=3, stride=2, pad=1, mode=mode))
for mode in (0, 2):
    for tag, w in (("window", 32), ("gather", 34)):
        _add(f"stem3x3_u8_{tag}_m{mode}", _u8(2, 3, 24, w, 40, k=3, stride=2, pad=1, mode=mode))
        _add(f"stem7x7_u8_{tag}_m{mode}", _u8(2, 3, 30, w, 24, k=7, stride=2, pad=3, mode=mode))
    for tag, s, oc in (("window", 1, 40), ("gather", 2, 240), ("window_s2", 2, 224)):
        _add(f"nhwc16_3x3_u8_{tag}_m{mode}", _u8(2, 16, 15, 17, oc, k=3, stride=s, pad=1, mode=mode))
    _add(f"nhwc32_3x3_u8_window_m{mode}", _u8(2, 32, 18, 18, 40, k=3, stride=2, pad=1, mode=mode))
# ---- CUDA-core kernels: depthwise (TMA int8, generic), direct, stem ----
for mode in (0, 1, 2):
    for s in (1, 2):
        _add(f"dw3x3_i8_s{s}_m{mode}", _i8(2, 64, 17, 19, 64, k=3, stride=s, pad=1, group=64, mode=mode))
    _add(f"direct3x3_i8_m{mode}", _i8(2, 16, 13, 15, 24, k=3, pad=1, mode=mode), flags=abi.PRERUN_NO_TENSORCORE)
    _add(f"stem_cc_i8_m{mode}", _i8(2, 3, 21, 23, 24, k=3, stride=2, pad=1, mode=mode), flags=abi.PRERUN_NO_TENSORCORE)
for s in (1, 2):
    _add(f"dw3x3_u8_s{s}", _u8(2, 64, 17, 19, 64, k=3, stride=s, pad=1, group=64))
_add("direct3x3_u8", _u8(2, 16, 13, 15, 24, k=3, pad=1), flags=abi.PRERUN_NO_TENSORCORE)
_add("stem_cc_u8", _u8(2, 3, 21, 23, 24, k=3, stride=2, pad=1), flags=abi.PRERUN_NO_TENSORCORE)
_add("fc_cc_i8", lambda r: ties.int8_fc(r, 5, 512, 200), flags=abi.PRERUN_NO_TENSORCORE)
# ---- glue ops ----
PW_EXACT_SHAPE = (2, 8, 9, 11)
for u8 in (False, True):
    d = "u8" if u8 else "i8"
    for elt, en in ((abi.ELT_SUM, "sum"), (abi.ELT_PROD, "prod")):
        _add(f"eltwise_{en}_{d}_padlanes", lambda r, u=u8, e=elt: ties.eltwise(r, u, e, shape=(2, 24, 9, 11)))
        _add(f"eltwise_{en}_{d}_nopad", lambda r, u=u8, e=elt: ties.eltwise(r, u, e, shape=(2, 32, 9, 11)))
        # fewer than 16 channels: the literal per-element kernel (kernels_direct.cu launch_pointwise)
        _add(f"eltwise_{en}_{d}_pwexact", lambda r, u=u8, e=elt: ties.eltwise(r, u, e, shape=PW_EXACT_SHAPE))
    _add(f"leaky_relu_{d}_pwexact", lambda r, u=u8: ties.relu(r, u, 2, shape=PW_EXACT_SHAPE))
    _add(f"relu_{d}", lambda r, u=u8: ties.relu(r, u))
    _add(f"leaky_relu_{d}", lambda r, u=u8: ties.relu(r, u, 2))
    _add(f"avgpool2x2_{d}_fast", lambda r, u=u8: ties.pool(r, u, abi.POOL_AVG, 2, 2))
    _add(f"avgpool2x2p1_{d}_fast", lambda r, u=u8: ties.pool(r, u, abi.POOL_AVG, 2, 2, pad=1))
    _add(f"avgpool2x2p1_caffe_{d}_fast", lambda r, u=u8: ties.pool(r, u, abi.POOL_AVG, 2, 2, pad=1, caffe=1))
    _add(f"maxpool3x3s2_{d}_fast", lambda r, u=u8: ties.pool(r, u, abi.POOL_MAX, 3, 2, pad=1, scale_ratio=2))
    _add(f"global_avgpool_{d}", lambda r, u=u8: ties.pool(r, u, abi.POOL_AVG, 4, 4, global_pool=True, shape=(2, 64, 4, 4),
                                                        scale_ratio=0.25))
    _add(f"concat_{d}_lut", lambda r, u=u8: ties.concat(r, u))
    # 24 + 40 channels: the second input starts off a 16-channel boundary, so both take the byte-wise kernel
    _add(f"concat_{d}_seam", lambda r, u=u8: ties.concat(r, u, shape=(2, 24, 6, 7), c2=40))

# the deferred rare-path queue: tie-sparse (every M = 2^-8: the queue is used, never full) and tie-dense (every M = 2^-1: more than
# 4 x FIXQ_CAP guarded elements per CTA, so most of them take the full-queue inline fallback)
def _sparse(r):
    case = ties.int8_conv(r, 2, 64, 96, 96, 128, mode=1, m_exps=(8,))
    case.min_tie_frac = 0.002  # M = 2^-8: one accumulator in 256 is a tie, by design
    return case


_add("queue_sparse", _sparse)
_add("queue_dense", _i8(8, 64, 96, 96, 128, mode=0, m_exps=(1,)))
_add("queue_dense_u8", lambda r: ties.uint8_conv(r, 8, 64, 96, 96, 128, s_out=2.0 ** -6))


def build(name):
    b, flags = CASES[name]
    case = b(_rng(name))
    case.name = name
    return case, flags


def run_case(ctx, name):
    """Run case `name` on the device (every layer read back) and compare with the exact reference.  Returns a message or None."""
    from tengine_b200 import runtime as rt

    case, flags = build(name)
    g = case.g
    want, rs = ties.exact_run(g, case.inputs)
    out = g.outputs[0]
    ties.check_not_vacuous(case, rs[out])
    gr = rt.Graph(ctx, g, flags | abi.PRERUN_NO_GRAPH)
    try:
        outs = gr.run(case.inputs)
        got = {L["output"]: gr.read_tensor(L["output"]) for L in g.layers}
        kernels = gr.layer_kernels()
    finally:
        gr.close()
    for li, L in enumerate(g.layers):
        t = L["output"]
        bad = got[t] != want[t]
        if bad.any():
            tie = rs[t].tie_mask()
            return (f"{name}: layer {li} ({kernels[li]}) differs from the exact reference in {int(bad.sum())} of {bad.size} bytes, "
                    f"{int((bad & tie).sum())} of them at exact ties; first at {np.argwhere(bad)[0].tolist()}")
    if not np.array_equal(outs[0], want[out]):
        return f"{name}: graph output differs from the last layer's tensor"
    return None


@pytest.mark.parametrize("name", list(CASES))
def test_tie_dense_layer(ctx, name):
    msg = run_case(ctx, name)
    assert msg is None, msg


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith(("stem3x3_i8_window", "nhwc16", "igemm_i8_outmode1", "dw3x3_i8_s1"))][:6])
def test_tie_dense_layer_against_oracle(ctx, oracle, name):
    """The small cases once more against the oracle (itself pinned to the exact reference on the CPU)."""
    from tengine_b200 import runtime as rt

    case, flags = build(name)
    gr = rt.Graph(ctx, case.g, flags)
    got = gr.run(case.inputs)[0]
    gr.close()
    assert np.array_equal(got, oracle.run(case.g, case.inputs, uint8_mode=0)[case.g.outputs[0]])


def _guarded_per_cta(case, sms):
    """Guarded elements (exact ties, clamped or not: the guard looks at t before the clamp) of every CTA of the persistent GEMM,
    from the exact t and the kernel's tile schedule (m-tile i of 128 rows goes to CTA i % grid; one N tile, one m-tile a stage)."""
    _, rs = ties.exact_run(case.g, case.inputs)
    t = rs[case.g.outputs[0]]
    tie = t.tie_mask()  # n, oc, h, w
    per_row = tie.transpose(0, 2, 3, 1).reshape(-1, tie.shape[1]).sum(1)
    m_tiles = (per_row.size + 127) // 128
    per_tile = np.add.reduceat(per_row, np.arange(0, per_row.size, 128))
    grid = min(m_tiles, sms)
    return np.bincount(np.arange(m_tiles) % grid, weights=per_tile, minlength=grid)


def test_queue_cases_reach_their_regimes():
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dense = _guarded_per_cta(build("queue_dense")[0], sms)
    assert dense.min() > 4 * FIXQ_CAP, (dense.min(), 4 * FIXQ_CAP)
    dense_u8 = _guarded_per_cta(build("queue_dense_u8")[0], sms)
    assert dense_u8.min() > 4 * FIXQ_CAP, (dense_u8.min(), 4 * FIXQ_CAP)
    sparse = _guarded_per_cta(build("queue_sparse")[0], sms)
    assert 0 < sparse.max() < FIXQ_CAP and sparse.sum() > 100, (sparse.min(), sparse.max())


# ---- instantiation coverage ----
def _expected_instantiations():
    exp = set()
    for u8, modes in ((0, (0, 1, 2)), (1, (0, 2))):
        for m in modes:
            for cs in (1, 2):
                for border in ((0,) if not u8 else (0, 1)):
                    exp.add(f"gemm_i8_tcgen05_kernel<U8={u8},MODE={m},CS={cs},BORDER={border}>")
        for m in modes:
            for k in (3, 7):
                exp.add(f"conv_gather_tc_kernel<MODE={m},U8={u8},KHW={k}>")
            for ly in (0, 1, 2, 3):
                exp.add(f"conv_window_tc_kernel<MODE={m},U8={u8},LAYOUT={ly}>")
    for k in ("conv_dw3x3_tma_pack3_kernel", "conv_dw3x3_tma_kernel<4,2>"):
        for m in (0, 1, 2):
            exp.add(f"{k} MODE={m}")
    return exp


def test_every_compiled_instantiation_is_launched():
    """All cases in one child process with TB200_DEBUG_LAUNCH: every instantiation the library compiles appears in its report, and
    each *_gather_* / *_window_* case launched only the kernel its name says."""
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_requant_ties"] + list(CASES), cwd=ROOT,
                       env=dict(os.environ, TB200_DEBUG_LAUNCH="1"), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    launched, per_case, cur = set(), {}, None
    for line in r.stderr.splitlines():
        if line.startswith(MARK):
            cur = line[len(MARK):].strip()
            continue
        m = re.match(r"tengine_b200: launch (\S+(?: MODE=\d)?)", line)
        if m:
            launched.add(m.group(1))
            per_case.setdefault(cur, set()).add(m.group(1))
    missing = sorted(_expected_instantiations() - launched)
    print("launched:", sorted(launched))
    assert not missing, f"never launched: {missing}"
    bad = []
    for name in CASES:
        for tag, kernel in (("_gather_", "conv_gather_tc_kernel<"), ("_window_", "conv_window_tc_kernel<")):
            got = per_case.get(name, set())
            if tag in name and (not got or any(not k.startswith(kernel) for k in got)):
                bad.append(f"{name}: launched {sorted(got)}")
    assert not bad, "\n".join(bad)


# ---- the literal-arithmetic kernel entry points (tb200k_*) on tie-dense layers: the control, pad lanes included ----
# tb200k_gemm_i8 passes the GEMM no rare-path queue
@pytest.mark.parametrize("name", ["direct3x3_i8_m1", "direct3x3_u8", "dw3x3_i8_s1_m1", "dw3x3_i8_s2_m0", "dw3x3_u8_s2", "gemm1x1_i8_m0_cs2",
                                  "fc_i8_m0"])
def test_tb200k_entry_points(ctx, name):
    import torch

    from tengine_b200 import runtime as rt
    from tests.test_gpu_kernel_abi import _cpad, _dev, _epilogue, _finish, _nhwc, _shape

    case, _ = build(name)
    g = case.g
    L = g.layers[0]
    want, _ = ties.exact_run(g, case.inputs)
    want = want[g.outputs[0]]
    x = case.inputs[0]
    n, c, h, w = x.shape
    oc = g.dims(g.outputs[0])[1]
    cp, ocp = _cpad(c), _cpad(oc)
    k = L["kernel_h"]
    keep = []
    e = _epilogue(g, L, keep)
    sh = _shape(g, L)
    lib = rt.lib()
    if k == 1:  # 1x1 conv or FC over a 1x1 input: the persistent GEMM, rows = pixels, K = cp
        wp = np.zeros((ocp, cp), g.np_dtype)
        wp[:oc, :c] = L["weight"].reshape(oc, c)
        fn, args = lib.tb200k_gemm_i8, (C.c_int64(n * h * w), cp, oc)
    elif L["group"] == 1:
        wp = np.zeros((ocp, k, k, cp), g.np_dtype)
        wp[:oc, :, :, :c] = L["weight"].transpose(0, 2, 3, 1)
        fn, args = lib.tb200k_conv_direct, (C.byref(sh),)
    else:
        wp = np.zeros((3, 3, cp), g.np_dtype)
        wp[:, :, :c] = L["weight"].reshape(c, 3, 3).transpose(1, 2, 0)
        fn, args = lib.tb200k_conv_dw3x3, (C.byref(sh),)
    din, dwt = _dev(_nhwc(x, cp)), _dev(wp)
    out = torch.full((n * sh.oh * sh.ow * ocp,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = fn(C.c_void_p(din.data_ptr()), C.c_void_p(dwt.data_ptr()), C.c_void_p(out.data_ptr()), *args, C.byref(e), C.c_void_p(ctx.stream))
    assert rc == 0, lib.tb200_last_error().decode()
    _finish(out.view(torch.uint8 if g.data_type == abi.DT_UINT8 else torch.int8), g, want)


def _main(names):
    from tengine_b200 import runtime as rt

    ctx = rt.Context(0)
    fails = 0
    try:
        for name in names:
            sys.stderr.write(MARK + name + "\n")
            sys.stderr.flush()
            msg = run_case(ctx, name)
            print(("FAIL " + msg) if msg else ("ok " + name), flush=True)
            fails += msg is not None
    finally:
        ctx.close()
    return 1 if fails else 0


if __name__ == "__main__":
    sys.exit(_main(sys.argv[1:]))
