"""TEST INFRASTRUCTURE: what the classification examples do with the graph's output tensor, restated -- the checker of
tb200_graph_topk / tb200k_class_topk.

examples/tm_classification_int8.c:163-164 dequantises with (float)q * scale, examples/tm_classification_uint8.c:169-170 with
((float)q - (float)zero_point) * scale, and both call print_topk(output_data, output_size, 5)
(examples/common/tengine_operations.c:1021-1038): ids 0..E-1 in buffer order, sort_cls_score (:991-1019) over the whole array,
entries 0..k-1 printed.  sort_cls_score is a first-element-pivot quicksort whose scans pass over equal scores, so it is unstable and
its tie order is part of the result.  Pinned against the example compiled as it is by tests/test_topk_pinned.py."""
import numpy as np


def dequantise(q, scale, zero_point, u8):
    """The examples' dequantisation in float32 arithmetic, one rounding per element.  The int8 example ignores the zero point."""
    q = np.asarray(q)
    f = q.astype(np.float32)
    with np.errstate(all="ignore"):
        if u8:
            f = f - np.float32(zero_point)
        return (f * np.float32(scale)).astype(np.float32)


def sort_cls_score(score, ids, left, right):
    """sort_cls_score(array, left, right) on the parallel lists `score` / `ids`, in place.  The body is the example's, line for line;
    its two recursive calls work on disjoint ranges, so they are taken from an explicit stack (all-equal scores would otherwise nest
    E deep)."""
    stack = [(left, right)]
    while stack:
        left, right = stack.pop()
        i, j = left, right
        if left >= right:
            continue
        key_s, key_i = score[left], ids[left]
        while left < right:
            while left < right and key_s >= score[right]:
                right -= 1
            score[left], ids[left] = score[right], ids[right]
            while left < right and key_s <= score[left]:
                left += 1
            score[right], ids[right] = score[left], ids[left]
        score[left], ids[left] = key_s, key_i
        stack.append((left + 1, j))
        stack.append((i, left - 1))


def sorted_classes(scores):
    """(scores [E] float32, ids [E] int32): the array print_topk holds after its sort, for one image's dequantised scores."""
    s = [float(v) for v in np.asarray(scores, np.float32).reshape(-1)]
    ids = list(range(len(s)))
    sort_cls_score(s, ids, 0, len(s) - 1)
    return np.array(s, np.float32), np.array(ids, np.int32)


def topk(q_nchw, scale, zero_point, u8, k):
    """q_nchw: [N, ...] quantised output in NCHW order; the classes of image i are its elements in that order.  Returns
    (scores [N, k] float32, ids [N, k] int32), entry r being entry r of the example's sorted array."""
    q = np.asarray(q_nchw)
    q = q.reshape(q.shape[0], -1)
    assert 1 <= k <= q.shape[1], (k, q.shape)
    scores, ids = np.empty((q.shape[0], k), np.float32), np.empty((q.shape[0], k), np.int32)
    for n in range(q.shape[0]):
        s, i = sorted_classes(dequantise(q[n], scale, zero_point, u8))
        scores[n], ids[n] = s[:k], i[:k]
    return scores, ids
