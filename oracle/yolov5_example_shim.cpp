// TEST INFRASTRUCTURE (oracle): the detection post-processing of the UNMODIFIED reference example examples/tm_yolov5s.cpp, compiled
// from the source where it lies (its main() is renamed, the C++ OpenCV it needs is replaced by oracle/cvstub) and exported through
// one C function, so that oracle/yolov5_post.py -- the checker of tb200_graph_yolov5_detect -- is pinned against the example's own
// code instead of a reading of it.  Built by oracle/build_yolov5_example.py into oracle/_ref/libyolov5_example.so.
#include <float.h>
#include <algorithm>
#include <cmath>
#include <vector>

#include <opencv2/core/core.hpp>

#include "common.h"
#include "tengine/c_api.h"
#include "tengine_operations.h"

// The image-loading code of this example names three things the YOLOv3-tiny example does not, and that oracle/cvstub (shared with
// oracle/yolo_example_shim.cpp) therefore lacks: a Mat(rows, cols, type, Scalar) constructor, copyMakeBorder and BORDER_CONSTANT.
// That code is never executed here; these stand-ins only let it compile, and carry no semantics.
namespace cv {
enum { BORDER_CONSTANT = 0 };
struct MatV5 : Mat
{
    MatV5() {}
    MatV5(const Mat& m) : Mat(m) {}
    MatV5(int, int, int, const Scalar&) {}
};
static inline void copyMakeBorder(const Mat&, Mat&, int, int, int, int, int, const Scalar&) {}
} // namespace cv

#define Mat MatV5
#define main tm_yolov5s_example_main
#include "tm_yolov5s.cpp"
#undef main
#undef Mat

// p8 / p16 / p32: the three float head tensors of ONE image in the layout the example indexes (:167), feat[a][h][w][85], with
// letterbox_rows x letterbox_cols the network input (each head is letterbox / stride cells).  The call sequence is main():561-576.
// Returns the number of kept boxes, written as (x, y, w, h, prob, label) rows.
extern "C" int yolov5_example_postprocess(const float* p8, const float* p16, const float* p32, int letterbox_rows, int letterbox_cols, float prob_threshold,
                                          float nms_threshold, float* out6, int max_out)
{
    std::vector<Object> proposals, objects8, objects16, objects32;
    generate_proposals(32, p32, prob_threshold, objects32, letterbox_cols, letterbox_rows);
    proposals.insert(proposals.end(), objects32.begin(), objects32.end());
    generate_proposals(16, p16, prob_threshold, objects16, letterbox_cols, letterbox_rows);
    proposals.insert(proposals.end(), objects16.begin(), objects16.end());
    generate_proposals(8, p8, prob_threshold, objects8, letterbox_cols, letterbox_rows);
    proposals.insert(proposals.end(), objects8.begin(), objects8.end());
    qsort_descent_inplace(proposals);
    std::vector<int> picked;
    nms_sorted_bboxes(proposals, picked, nms_threshold);
    int n = 0;
    for (size_t i = 0; i < picked.size() && n < max_out; i++, n++)
    {
        const Object& o = proposals[picked[i]];
        float* r = out6 + 6 * n;
        r[0] = o.rect.x, r[1] = o.rect.y, r[2] = o.rect.width, r[3] = o.rect.height, r[4] = o.prob, r[5] = (float)o.label;
    }
    return (int)picked.size();
}

extern "C" float yolov5_example_sigmoid(float x) { return sigmoid(x); }
