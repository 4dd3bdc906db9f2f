"""CPU restatement of the detection post-processing of examples/tm_yolov5s.cpp (TEST INFRASTRUCTURE; checker of
tb200_graph_yolov5_detect): dequantisation ((float)q - zp) * scale, generate_proposals (:140-207), then the same
qsort_descent_inplace (:61-104) and nms_sorted_bboxes (:106-138) as examples/tm_yolov3_tiny_uint8.cpp, shared with
oracle/yolo_post.py.  The proposal sequence is main():561-576: heads in the order given (the example's is stride 32, 16, 8).

Layout: the heads are the raw [N, 3 * (5 + classes), H, W] outputs of the three 1x1 detection convolutions.  The example indexes
feat[a][h][w][k] (:167, after the Reshape / Transpose of the ONNX graph), which is channel a * (5 + classes) + k at (h, w) here.

PINNED: tests/test_yolov5_post_pinned.py compares this file, box for box and bit for bit, with the example's own functions compiled
from the unmodified source (oracle/yolov5_example_shim.cpp, built into oracle/_ref/libyolov5_example.so) and with a committed fixture
of their output.  The example's sigmoid is the same float-expf form as the YOLOv3-tiny example's (pinned there too).
"""
import numpy as np

from oracle.yolo_post import _sigmoid, nms_sorted_bboxes, qsort_descent_inplace

f32 = np.float32
ANCHORS = [10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326]  # tm_yolov5s.cpp:143
# (stride, anchors6) in the example's proposal order; anchors[(anchor_group - 1) * 6 + ...] with group 3 / 2 / 1 for stride 32 / 16 / 8
HEADS_BY_STRIDE = {32: ANCHORS[12:18], 16: ANCHORS[6:12], 8: ANCHORS[0:6]}


def generate_proposals(stride, feat, anchors6, num_classes, prob_threshold):
    """feat: dequantised [3*(5+cls), H, W] float32 of ONE image.  Returns [(x, y, w, h, prob, label)] in the example's order."""
    _, fh, fw = feat.shape
    out = []
    per = num_classes + 5
    st = f32(stride)
    for h in range(fh):
        for w in range(fw):
            for a in range(3):
                scores = feat[a * per + 5:a * per + 5 + num_classes, h, w]
                cls = int(np.argmax(scores))  # first maximum == the example's strict `>` scan
                final = f32(_sigmoid(feat[a * per + 4, h, w]) * _sigmoid(scores[cls]))
                if final >= f32(prob_threshold):
                    dx, dy, dw, dh = (_sigmoid(feat[a * per + k, h, w]) for k in range(4))
                    pred_cx = f32(f32(f32(f32(dx * f32(2.0)) - f32(0.5)) + f32(w)) * st)  # (dx * 2.0f - 0.5f + w) * stride
                    pred_cy = f32(f32(f32(f32(dy * f32(2.0)) - f32(0.5)) + f32(h)) * st)
                    pred_w = f32(f32(f32(dw * dw) * f32(4.0)) * f32(anchors6[2 * a]))  # dw * dw * 4.0f * anchor_w
                    pred_h = f32(f32(f32(dh * dh) * f32(4.0)) * f32(anchors6[2 * a + 1]))
                    x0, y0 = f32(pred_cx - f32(pred_w * f32(0.5))), f32(pred_cy - f32(pred_h * f32(0.5)))
                    x1, y1 = f32(pred_cx + f32(pred_w * f32(0.5))), f32(pred_cy + f32(pred_h * f32(0.5)))
                    out.append([x0, y0, f32(x1 - x0), f32(y1 - y0), final, cls])
    return out


def detect(outputs, scales, zeros, heads, num_classes, prob_threshold, nms_threshold):
    """outputs: per head a quantised NCHW array [N, 3*(5+cls), H, W] (uint8 or int8); heads: [(output index, stride, anchors6)] in
    proposal order.  Returns per image the kept boxes [(x, y, w, h, prob, label)]."""
    n = outputs[0].shape[0]
    res = []
    for img in range(n):
        props = []
        for (oi, stride, anchors6) in heads:
            q = outputs[oi][img].astype(np.float32)
            feat = ((q - f32(zeros[oi])) * f32(scales[oi])).astype(np.float32)
            props += generate_proposals(stride, feat, anchors6, num_classes, prob_threshold)
        if props:
            qsort_descent_inplace(props, 0, len(props) - 1)
        res.append([props[i] for i in nms_sorted_bboxes(props, nms_threshold)])
    return res
