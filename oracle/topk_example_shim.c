// TEST INFRASTRUCTURE (oracle): the ranking step of the UNMODIFIED reference examples, print_topk of
// examples/common/tengine_operations.c, callable without its fprintf.  That file is compiled from where it lies by including it, so
// that its static sort_cls_score is reachable; oracle/topk.py -- the checker of tb200_graph_topk -- is pinned against it instead of
// a reading of it.  Built by oracle/build_topk_example.py into oracle/_ref/libtopk_example.so.
#include "tengine_operations.c"

// Fills the array as print_topk does (id = position, score = data[position]), sorts it with the example's own function and returns
// all of it: ids[0..total_num), scores[0..total_num).
__attribute__((visibility("default"))) int topk_example_sorted(const float* data, int total_num, int* ids, float* scores)
{
    cls_score* cls_scores = (cls_score*)malloc(total_num * sizeof(cls_score));
    if (!cls_scores) return -1;
    for (int i = 0; i < total_num; i++)
    {
        cls_scores[i].id = i;
        cls_scores[i].score = data[i];
    }
    sort_cls_score(cls_scores, 0, total_num - 1);
    for (int i = 0; i < total_num; i++)
    {
        ids[i] = cls_scores[i].id;
        scores[i] = cls_scores[i].score;
    }
    free(cls_scores);
    return 0;
}
