// TEST INFRASTRUCTURE (oracle): the input preprocessing of the UNMODIFIED reference examples examples/tm_classification_int8.c and
// examples/tm_classification_uint8.c, compiled from the sources where they lie (their main(), tengine_classify() and show_usage()
// are renamed so that both fit in one library) and linked with examples/common/tengine_operations.c, so that oracle/image_pre.py --
// the checker of tb200_graph_upload_images -- is pinned against the examples' own code instead of a reading of it.  Built by
// oracle/build_image_example.py into oracle/_ref/libimage_example.so, which exports, unchanged:
//   get_input_int8_data(image_file, int8_t* out, img_h, img_w, float* mean, float* scale, float input_scale)
//   get_input_uint8_data(image_file, uint8_t* out, img_h, img_w, float* mean, float* scale, float input_scale, int zero_point)
//   stbi_load / stbi_image_free (the decoder the examples read files with) and stbi_write_png (to write RGBA test images).
#define main tm_classification_int8_main
#define tengine_classify tm_classification_int8_classify
#define show_usage tm_classification_int8_show_usage
#include "tm_classification_int8.c"
#undef main
#undef tengine_classify
#undef show_usage

#define main tm_classification_uint8_main
#define tengine_classify tm_classification_uint8_classify
#define show_usage tm_classification_uint8_show_usage
#include "tm_classification_uint8.c"
#undef main
#undef tengine_classify
#undef show_usage
