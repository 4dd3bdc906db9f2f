"""Pins oracle/topk.py -- the checker of tb200_graph_topk / tb200k_class_topk -- against the ranking step of the UNMODIFIED
classification examples (print_topk and its sort_cls_score, examples/common/tengine_operations.c): (a) the committed fixture
tests/golden/topk_example.npz, the example's whole sorted array per case (generator: tests/golden/make_golden_topk.py), everywhere;
(b) the compiled example itself, live, on seeded outputs, where oracle/_ref/libtopk_example.so exists.  Ids and score bits.  Also: a
Python model of the device algorithm (pruned replay, 32 positions per scan step) equals the full sort on the reported positions, and
abi.ClassScore has the layout of tb200_class_score."""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import topk  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "topk_example.npz")


def _case(d, k):
    s, zp, u8 = d[f"quant_{k}"]
    return d[f"q_{k}"], np.float32(s), int(zp), bool(u8)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_restatement_equals_the_committed_output_of_the_unmodified_example():
    d = np.load(FIXTURE)
    names = list(d["names"])
    assert len(names) >= 25
    for k, name in enumerate(names):
        q, s, zp, u8 = _case(d, k)
        assert q.dtype == (np.uint8 if u8 else np.int8), name
        scores, ids = topk.topk(q[None], s, zp, u8, q.size)
        assert np.array_equal(ids[0], d[f"ids_{k}"]), name
        assert np.array_equal(_bits(scores[0]), _bits(d[f"scores_{k}"])), name
        assert sorted(ids[0].tolist()) == list(range(q.size)), name
    assert {int(d[f"q_{k}"].size) for k in range(len(names))} >= {1, 2, 5, 33, 1000, 1001}
    assert {int(d[f"quant_{k}"][1]) for k in range(len(names)) if d[f"quant_{k}"][2]} >= {0, 3, 128}
    assert any(d[f"quant_{k}"][0] < 0 for k in range(len(names))) and any(d[f"quant_{k}"][0] == 0 for k in range(len(names)))


def _stable_order(scores, ascending_ids):
    """Descending score, ties by ascending (or descending) id: what a stable top-k with either tie rule reports."""
    idx = np.arange(scores.size)
    return np.lexsort((idx if ascending_ids else -idx, -scores.astype(np.float64)))


# case -> the k at which a stable top-k already differs (one flat block of equal peaks comes out in descending id at first)
TIED = {"two_values_int8": 5, "two_values_uint8_zp128": 5, "softmax_like_int8": 5, "softmax_like_uint8_zp0": 5, "softmax_like_flat_int8": 64,
        "narrow_random_int8": 5, "coarse_zero_point_uint8": 5}


def test_the_fixture_reaches_the_tie_orders_it_is_there_for():
    d = np.load(FIXTURE)
    names = list(d["names"])
    for name, n in TIED.items():
        k = names.index(name)
        q, s, zp, u8 = _case(d, k)
        f = topk.dequantise(q, s, zp, u8)
        assert len(np.unique(f)) < f.size / 4, name  # distinct bytes may share a float: ties are counted on the scores
        top = d[f"ids_{k}"][:n]
        assert not np.array_equal(top, _stable_order(f, True)[:n]), name
        assert not np.array_equal(top, _stable_order(f, False)[:n]), name
    # with every score equal no scan finds anything to move: the example leaves the classes in id order
    for name in ("all_equal_int8", "all_equal_uint8_zp3", "underflowing_scale_int8"):
        k = names.index(name)
        assert np.array_equal(d[f"ids_{k}"], np.arange(d[f"q_{k}"].size)), name
    # distinct scores leave no choice
    for name in ("ascending_int8", "descending_uint8_zp128", "negative_scale_int8"):
        k = names.index(name)
        q, s, zp, u8 = _case(d, k)
        f = topk.dequantise(q, s, zp, u8)
        if len(np.unique(f)) == f.size:
            assert np.array_equal(d[f"ids_{k}"], _stable_order(f, True)), name
    k = names.index("underflowing_scale_int8")
    assert set(_bits(d[f"scores_{k}"]).tolist()) == {0, 0x80000000}  # +0 and -0: equal scores with different bits
    k = names.index("overflowing_scale_int8")
    assert np.isinf(d[f"scores_{k}"]).any() and not np.isnan(d[f"scores_{k}"]).any()


def test_restatement_equals_the_compiled_example_live():
    import make_golden_topk as gen

    if not os.path.exists(gen.LIB):
        pytest.skip("oracle/_ref/libtopk_example.so absent (built by oracle/build_topk_example.py where the reference tree exists)")
    L = gen.example_lib()
    rng = np.random.default_rng(2024)
    for trial in range(300):
        e = int(rng.integers(1, 400)) if trial % 10 else 1000
        u8 = bool(trial % 2)
        spread = int(rng.choice([1, 2, 4, 16, 256]))
        q = rng.integers(0, spread, e) + (0 if u8 else -(spread // 2))
        q = q.astype(np.uint8 if u8 else np.int8)
        if trial % 7 == 0:
            q = np.sort(q)[::int(rng.choice([-1, 1]))].copy()
        s = np.float32(rng.choice([0.0213, -0.0471, 0.0, 1.0]))
        zp = int(rng.integers(0, 256)) if u8 else 0
        f = topk.dequantise(q, s, zp, u8)
        want_s, want_i = gen.run_example(L, f)
        got_s, got_i = topk.topk(q[None], s, zp, u8, e)
        assert np.array_equal(got_i[0], want_i), (trial, e, u8, spread)
        assert np.array_equal(_bits(got_s[0]), _bits(want_s)), (trial, e, u8, spread)


def device_model(scores, k):
    """The device algorithm on one image's scores: sort_cls_score with (a) a right-hand sub-range that starts at or beyond k dropped,
    the others kept on a stack, the left one continued with at once; (b) every scan taking 32 positions per step and the nearest
    position where the example's comparison fails.  Returns (scores, ids) of positions 0..k-1 and the deepest the stack got."""
    s = [float(v) for v in np.asarray(scores, np.float32)]
    ids = list(range(len(s)))
    pending, deepest = [], 0
    i, j = 0, len(s) - 1
    while True:
        if i >= j:
            if not pending:
                break
            i, j = pending.pop()
            continue
        left, right = i, j
        key, key_id = s[left], ids[left]
        while left < right:
            while left < right:
                stop = [lane for lane in range(32) if right - lane > left and not key >= s[right - lane]]
                if stop:
                    right -= stop[0]
                    break
                right = max(left, right - 32)
            s[left], ids[left] = s[right], ids[right]
            while left < right:
                stop = [lane for lane in range(32) if left + lane < right and not key <= s[left + lane]]
                if stop:
                    left += stop[0]
                    break
                left = min(right, left + 32)
            s[right], ids[right] = s[left], ids[left]
        s[left], ids[left] = key, key_id
        if left + 1 < k and left + 1 < j:
            pending.append((left + 1, j))
            deepest = max(deepest, len(pending))
        j = left - 1
    return np.array(s[:k], np.float32), np.array(ids[:k], np.int32), deepest


def test_pruned_parallel_replay_equals_the_full_sort_on_the_reported_positions():
    d = np.load(FIXTURE)
    names = list(d["names"])
    for k_case, name in enumerate(names):
        q, s, zp, u8 = _case(d, k_case)
        f = topk.dequantise(q, s, zp, u8)
        for k in sorted({1, 5, 64, q.size}):
            if k > q.size or (k == q.size and q.size > 300 and k_case % 4):  # the unpruned run of a 1000-class case is slow in Python
                continue
            got_s, got_i, deepest = device_model(f, k)
            assert np.array_equal(got_i, d[f"ids_{k_case}"][:k]), (name, k)
            assert np.array_equal(_bits(got_s), _bits(d[f"scores_{k_case}"][:k])), (name, k)
            assert deepest <= k, (name, k, deepest)


def test_class_score_struct_matches_header():
    from tengine_b200 import abi

    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "tengine_b200.h"\nint main(){printf("%zu %zu %zu %d %d\\n", sizeof(tb200_class_score), '
           'offsetof(tb200_class_score, score), offsetof(tb200_class_score, id), TB200_TOPK_MAX, TB200_TOPK_MAX_CLASSES);return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")]).split()
    assert [int(x) for x in out] == [ctypes.sizeof(abi.ClassScore), abi.ClassScore.score.offset, abi.ClassScore.id.offset, abi.TOPK_MAX, abi.TOPK_MAX_CLASSES]
