// engine.cu -- the C ABI of include/tengine_b200.h: context, subgraph planner/executor, weight pre-packing.
//
// One tb200_graph is what the Tengine device glue stores in subgraph->device_graph.  prerun = the analogue of
// the CPU device's create_exec_graph + alloc_exec_graph_mem + prerun_exec_graph (source/device/cpu/
// cpu_device.c:62-95) and of conv_hcl_prerun's weight packing (conv_kernel_x86.c:2137-2209); run = the
// analogue of cpu_device.c:97-221 with every node executing on the GPU.  No CPU compute path exists here.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tengine_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace tb200;

#define TB200_OP_NOP_ (-1)  // planner-internal: a node folded into its producer
#define TB200_OP_LUT2_ (-2) // planner-internal: Sigmoid + Eltwise-PROD with the Sigmoid's input, as one byte table
#define TB200_PACK_FORMAT 5  // bump whenever the layout or content of the packed weight arena changes (pack cache key)

// ---- packed-weight cache directory (SURVEY.md 8(f)-3): tb200_pack_cache_dir() or the environment ----
static std::string g_pack_cache_dir;
static bool g_pack_cache_set = false;
static std::string pack_cache_dir()
{
    if (g_pack_cache_set) return g_pack_cache_dir;
    const char* e = getenv("TG_B200_PACK_CACHE");
    return e ? std::string(e) : std::string();
}

// ---- error reporting -------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_OK(call)                                                                                       \
    do                                                                                                      \
    {                                                                                                       \
        cudaError_t _e = (call);                                                                            \
        if (_e != cudaSuccess) return fail(TB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// A registered (page-locked) range of caller memory: tb200_graph_run pins the application's NCHW buffers the first time it
// sees them (cudaHostRegister, portable across the group's GPUs) so that every later H2D / D2H copy is a true async DMA.
struct HostReg
{
    const uint8_t* p;
    size_t bytes;
    bool ours; // false: the range was already page-locked by the application (cudaHostAlloc / its own registration)
};

// One context per GPU.  A multi-GPU context (tb200_context_create_multi, SURVEY.md 8(e)) is the context of GPU 0 plus `peers`
// (GPUs 1..R-1), all driven by the calling thread; `comms` are the ncclComm_t of ncclCommInitAll over the group.
struct tb200_context
{
    int device;
    int num_sms;
    cudaStream_t stream;
    std::vector<tb200_context*> peers;
    std::vector<void*> comms; // [R] when NCCL is in use
    const char* bcast_kind = "none";
    std::vector<HostReg> host_regs;
    std::vector<const void*> host_reg_failed;
    void* fixq = nullptr; // scratch of the GEMM kernels' deferred rare path: FIXQ_CAP entries per SM (gemm_tcgen05.cu)
};
static constexpr int FIXQ_CAP = 4096;
// TB200_DEBUG_STAGES=1: progress lines of the multi-GPU set-up on stderr (which call a hang or an error sits in)
#define STAGE(...)                                                                  \
    do                                                                              \
    {                                                                               \
        static const bool on_ = getenv("TB200_DEBUG_STAGES") != nullptr;             \
        if (on_) fprintf(stderr, "tengine_b200 stage: " __VA_ARGS__), fputc('\n', stderr), fflush(stderr); \
    } while (0)

// ---- NCCL, loaded at run time (libnccl.so.2: the copy torch already mapped when running under Python, the system one
//      otherwise) so that single-GPU users never need it.  Only what the one broadcast at prerun needs. ----
struct NcclApi
{
    void* handle = nullptr;
    int (*CommInitAll)(void**, int, const int*) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
static NcclApi* nccl_api()
{
    static NcclApi api;
    static bool tried = false;
    if (tried) return api.ok ? &api : nullptr;
    tried = true;
    if (getenv("TB200_NO_NCCL")) return nullptr;
    // TB200_NCCL_LIB names the copy to use; else whatever "libnccl.so.2" resolves to -- a copy the process has already mapped (the one
    // torch bundles, when running under Python: tengine_b200/runtime.py maps it first on purpose) or the system one
    const char* forced = getenv("TB200_NCCL_LIB");
    if (forced && *forced) api.handle = dlopen(forced, RTLD_NOW | RTLD_GLOBAL);
    for (const char* name : {"libnccl.so.2", "libnccl.so"})
        if (!api.handle) api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) return nullptr;
    api.CommInitAll = (int (*)(void**, int, const int*))dlsym(api.handle, "ncclCommInitAll");
    api.CommDestroy = (int (*)(void*))dlsym(api.handle, "ncclCommDestroy");
    api.GroupStart = (int (*)())dlsym(api.handle, "ncclGroupStart");
    api.GroupEnd = (int (*)())dlsym(api.handle, "ncclGroupEnd");
    api.Broadcast = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(api.handle, "ncclBroadcast");
    api.GetErrorString = (const char* (*)(int))dlsym(api.handle, "ncclGetErrorString");
    api.ok = api.CommInitAll && api.CommDestroy && api.GroupStart && api.GroupEnd && api.Broadcast && api.GetErrorString;
    return api.ok ? &api : nullptr;
}

enum StepKind
{
    K_NCHW2NHWC,
    K_NHWC2NCHW,
    K_CONV_STEM,
    K_GATHER_TC,
    K_CONV_DW,
    K_CONV_DIRECT,
    K_GEMM,
    K_IGEMM,
    K_POOL,
    K_POINTWISE,
    K_CONCAT_PART,
    K_UPSAMPLE,
    K_COPY,
    K_LUT,
    K_SOFTMAX,
    K_RESHAPE,
    K_NONE // a node folded into its producer
};
static const char* kStepName[] = {"nchw_to_nhwc", "nhwc_to_nchw", "conv_stem_nchw_dp4a", "conv_gather_tcgen05", "conv_dw_direct", "conv_direct_dp4a",
                                  "gemm_i8_tcgen05", "conv_igemm_i8_tcgen05", "pool", "pointwise", "concat_requant", "upsample_nearest", "copy",
                                  "byte_lut", "softmax", "reshape_nchw_order", "fused_into_producer"};

struct Step
{
    int kind;
    int layer; // -1 for layout steps
    const void* in = nullptr;
    const void* in2 = nullptr;
    const void* w = nullptr;
    void* out = nullptr;
    ConvShape cs{};
    PoolShape ps{};
    PointwiseParams pp{};
    EpiParams epi{};
    GemmPlan gemm{};
    const int32_t* btab = nullptr; // uint8 tensor-core kinds: padding-tap corrections
    DwPlan dwp{};
    WindowPlan wp{}; // K_GATHER_TC: TMA-staged input window (conv_window.cu) when applicable
    long long bytes = 0; // pointwise / copy
    // concat / layout
    long long npix = 0;
    int c = 0, cp_in = 0, cp_out = 0, c_off = 0, n = 0, h = 0, w_ = 0, scale = 0;
    int c_write = 0;             // concat: channels written from c_off (the last input also clears the pad lanes)
    int oc_ = 0, oh_ = 0, ow_ = 0; // reshape: output dims
    void* scratch = nullptr;     // reshape: NCHW-ordered staging
    int nhwc16 = 0; // K_GATHER_TC: the input is a 16-channel NHWC tensor (else the NCHW network input)
    float s_in = 0, s_out = 0;
    int z_in = 0, z_out = 0;
    bool u8 = false;
};

struct TensorInfo
{
    tb200_tensor_desc d;
    int cp;
    size_t nhwc_bytes, nchw_bytes;
    size_t off; // offset in the activation arena
    size_t slot_bytes = 0;
    int first_def = INT_MAX, last_use = -1; // liveness in layer order (arena slot reuse)
    uint8_t* dev = nullptr;
    int input_index = -1, output_index = -1;
    bool nhwc_needed = false; // graph inputs: a consumer needs the NHWC copy
    int producer = -1;
};

struct WeightBlob
{
    size_t w_off, bias_off, scale_off, fast_off, btab_off, w_size;
};

// Everything the planner decides for one layer.  plan_kernels fills in the kernel choice and what follows from it once,
// fuse_nodes and prove_fast_epilogues add their part; no later pass re-derives a decision from the descriptors.
struct LayerPlan
{
    int kind = K_NONE;
    WeightBlob blob{};       // where the layer's packed data sits in the weight arena
    bool reads_nchw = false; // stem kinds: the layer reads the NCHW graph input itself (no NHWC copy)
    int nhwc16 = 0;          // K_GATHER_TC over a 16- / 32-channel NHWC tensor
    bool u8_tc = false;      // uint8 K_GEMM / K_IGEMM / K_GATHER_TC: epilogue constants in the tensor-core layout
    int gemm_zp = 0;         // zero-point argument of the GEMM planners: 1 + weight zero point for uint8, else 0
    size_t k = 0;            // conv / FC: real K extent per output channel
    int fuse_bias = 0;       // the int8 fast epilogue folds the bias into its FMA (an int: the pack-cache key hashes it so)
    bool fast_ok = true;     // conv / FC: the fast epilogue is proven exact (fast-int proof and uint8 tensor-core proof)
    int post_relu = 0;       // eltwise: the folded ReLU that follows it
    int pool_relu = -1;      // max pooling: the folded (leaky) ReLU layer before it
    int silu_sig = -1;       // Eltwise-PROD turned byte table: the folded Sigmoid layer
    int silu_operand = 0;    // which operand of the product the sigmoid was (operand scales differ)
    size_t scratch_off = 0;  // K_RESHAPE: NCHW staging in the activation arena
};

// The launch sequences of one shard for one active batch: images [0, n) of the shard's arena as a whole and as pipeline chunks,
// and their CUDA graphs.  n == 0 (a shard left without images) has no steps at all.
struct BatchPlan
{
    int n = -1;
    std::vector<Step> steps;
    int chunks = 1;
    std::vector<int> chunk_first, chunk_count; // images of pipeline chunk k: [first, first + count)
    std::vector<std::vector<Step>> chunk_steps;
    std::vector<cudaGraph_t> cu_graphs; // [0] = whole slice, [1..K] = the pipeline chunks
    std::vector<cudaGraphExec_t> cu_execs;
    double work_ops = 0, work_bytes = 0, work_wbytes = 0;
    int num_launches = 0;
};

struct tb200_graph
{
    tb200_context* ctx;
    int flags;
    std::vector<TensorInfo> tensors;
    std::vector<tb200_layer_desc> layers;
    std::vector<const char*> layer_kernel;
    std::vector<LayerPlan> plan;
    std::vector<int> input_ids, output_ids;
    std::vector<uint8_t*> in_nchw_dev, out_nchw_dev;
    uint8_t* act_arena = nullptr;
    size_t act_bytes = 0;
    uint8_t* w_arena = nullptr;
    size_t w_bytes = 0;
    // tb200_graph_set_batch: `prepared` covers the batch of prerun, `other` the most recent smaller one; `cur` is the active one
    BatchPlan prepared, other;
    BatchPlan* cur = &prepared;
    int other_batch = 0; // the active batch `other` was built for (root; 0: none)
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_out;
    cudaEvent_t ev_done = nullptr;
    // batch sharding over the GPUs of a multi-GPU context: this graph is the shard of GPU 0 and owns the others.
    // first_image / num_images: the shard's part of the active batch (num_images may be 0); prep_images: its part of the batch
    // of prerun, the dim 0 of its tensors; total_images: that batch; batch: the active one (root)
    std::vector<tb200_graph*> shards;
    int first_image = 0, num_images = 0, prep_images = 0, total_images = 0, batch = 0;
    size_t act_unshared_bytes = 0; // what the arena would need without slot reuse (introspection)
    int pack_cache_state = 0;      // 0 no cache directory, 1 packed and written, 2 read from the cache
    // tb200_graph_upload_images: device copy of this shard's pixel span, its image descriptors (staged through page-locked host
    // memory that is rewritten only after img_ev, the previous descriptor copy, has completed); grown on demand
    uint8_t* img_stage = nullptr;
    size_t img_stage_bytes = 0;
    ImageDesc *img_desc = nullptr, *img_desc_host = nullptr;
    int img_desc_cap = 0;
    cudaEvent_t img_ev = nullptr;
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// 64-bit FNV-1a: the pack-cache key and the TB200_DEBUG_HASH lines.  `h` continues an earlier hash.
static const uint64_t kFnvBasis = 1469598103934665603ull;
static uint64_t fnv1a(const void* p, size_t n, uint64_t h = kFnvBasis)
{
    for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
    return h;
}

// ---- library / device ------------------------------------------------------------------------------------
extern "C" {

int tb200_abi_version(void) { return TB200_ABI_VERSION; }
const char* tb200_last_error(void) { return g_err; }

int tb200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess)
    {
        cudaGetLastError();
        return 0;
    }
    int good = 0;
    for (int i = 0; i < n; i++)
    {
        int major = 0;
        int minor = -1;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess &&
            cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, i) == cudaSuccess && major == 9 && minor == 0)
            good++;
    }
    return good;
}

static int context_create_one(int cuda_device, tb200_context** out)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
    {
        cudaGetLastError();
        return fail(TB200_ERR_NO_DEVICE, "no CUDA device visible: the H100 backend has no CPU fallback");
    }
    if (cuda_device < 0 || cuda_device >= n) return fail(TB200_ERR_INVALID, "cuda device %d out of range (%d)", cuda_device, n);
    int major = 0, minor = 0, sms = 0;
    CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, cuda_device));
    CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, cuda_device));
    CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cuda_device));
    if (major != 9 || minor != 0) return fail(TB200_ERR_NO_DEVICE, "device %d is sm_%d%d; this backend is built for sm_90a only", cuda_device, major, minor);
    CUDA_OK(cudaSetDevice(cuda_device));
    cudaStream_t st;
    CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    tb200_context* c = new tb200_context();
    c->device = cuda_device;
    c->num_sms = sms;
    c->stream = st;
    CUDA_OK(cudaMalloc(&c->fixq, (size_t)sms * FIXQ_CAP * 16));
    *out = c;
    return 0;
}

static void host_unregister_all(tb200_context* ctx)
{
    for (const HostReg& r : ctx->host_regs)
        if (r.ours && cudaHostUnregister((void*)r.p) != cudaSuccess) cudaGetLastError(); // the owner may have freed it already
    ctx->host_regs.clear();
    ctx->host_reg_failed.clear();
}

int tb200_context_create(int cuda_device, tb200_context** out)
{
    if (!out) return fail(TB200_ERR_INVALID, "null out");
    return context_create_one(cuda_device, out);
}

// SURVEY.md 8(e): one process drives R GPUs; the batch of every run is cut into R contiguous slices of dim 0.  The packed
// weight arena is built once (GPU 0) and reaches the other GPUs by ONE grouped ncclBroadcast at prerun (communicators from
// ncclCommInitAll); there is no collective in the steady state.  A device listed twice (tests on a one-GPU box) rules NCCL
// out (it refuses duplicate devices): the arena then travels by cudaMemcpyPeerAsync, everything else is identical.
int tb200_context_create_multi(const int* cuda_devices, int num_devices, tb200_context** out)
{
    if (!out || !cuda_devices || num_devices < 1 || num_devices > 64) return fail(TB200_ERR_INVALID, "bad device list");
    tb200_context* root = nullptr;
    int rc = context_create_one(cuda_devices[0], &root);
    if (rc) return rc;
    bool distinct = true;
    for (int i = 1; i < num_devices; i++)
    {
        tb200_context* p = nullptr;
        if ((rc = context_create_one(cuda_devices[i], &p)) != 0)
        {
            tb200_context_destroy(root);
            return rc;
        }
        root->peers.push_back(p);
        for (int j = 0; j < i; j++) distinct &= cuda_devices[j] != cuda_devices[i];
    }
    if (num_devices > 1)
    {
        root->bcast_kind = "memcpy_peer";
        NcclApi* nc = distinct ? nccl_api() : nullptr;
        if (nc)
        {
            std::vector<void*> comms(num_devices, nullptr);
            STAGE("ncclCommInitAll over %d devices ...", num_devices);
            const int r = nc->CommInitAll(comms.data(), num_devices, cuda_devices);
            STAGE("ncclCommInitAll -> %d", r);
            if (r == 0)
                root->comms = comms, root->bcast_kind = "nccl";
            else
                fprintf(stderr, "tengine_b200: ncclCommInitAll failed (%s); the weight arena will be broadcast with cudaMemcpyPeer\n", nc->GetErrorString(r));
        }
        else if (distinct && !getenv("TB200_NO_NCCL"))
            fprintf(stderr, "tengine_b200: libnccl.so.2 not found; the weight arena will be broadcast with cudaMemcpyPeer\n");
        cudaSetDevice(cuda_devices[0]);
    }
    *out = root;
    return 0;
}

int tb200_context_destroy(tb200_context* ctx)
{
    if (!ctx) return 0;
    host_unregister_all(ctx);
    if (!ctx->comms.empty())
        if (NcclApi* nc = nccl_api())
            for (void* c : ctx->comms)
                if (c) nc->CommDestroy(c);
    for (tb200_context* p : ctx->peers) tb200_context_destroy(p);
    cudaSetDevice(ctx->device);
    cudaStreamDestroy(ctx->stream);
    if (ctx->fixq) cudaFree(ctx->fixq);
    delete ctx;
    return 0;
}

void* tb200_context_stream(tb200_context* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int tb200_context_num_gpus(tb200_context* ctx) { return ctx ? 1 + (int)ctx->peers.size() : 0; }
static tb200_context* context_of(tb200_context* ctx, int index)
{
    if (!ctx || index < 0 || index > (int)ctx->peers.size()) return nullptr;
    return index == 0 ? ctx : ctx->peers[index - 1];
}
int tb200_context_gpu(tb200_context* ctx, int index)
{
    tb200_context* c = context_of(ctx, index);
    return c ? c->device : -1;
}
void* tb200_context_stream_of(tb200_context* ctx, int index)
{
    tb200_context* c = context_of(ctx, index);
    return c ? (void*)c->stream : nullptr;
}
const char* tb200_context_broadcast_kind(tb200_context* ctx) { return ctx ? ctx->bcast_kind : "none"; }

void* tb200_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess)
    {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void tb200_host_free(void* p)
{
    if (p) cudaFreeHost(p);
}

int tb200k_cpad(int channels) { return cpad(channels); }

} // extern "C"

// cudaMemcpyAsync between the device and pageable host memory: the caller's buffers and the library's own (the packed weight image, the
// detection tables).  host_pin keeps a caller buffer registered until postrun; once the caller frees it, a later allocation at that
// address -- a caller buffer of another size (a batch changed with tb200_graph_set_batch), or a vector of this library -- can start
// inside the stale registration and run past it, and CUDA refuses the copy (invalid argument).  Then every GPU of the group finishes
// its queued work, all of this context's registrations are dropped and the copy is issued once more; registrations come back as
// buffers are seen again.
static cudaError_t host_copy(tb200_context* root, void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st)
{
    cudaError_t e = cudaMemcpyAsync(dst, src, bytes, kind, st);
    if (e != cudaErrorInvalidValue || root->host_regs.empty()) return e;
    cudaGetLastError();
    int dev = 0;
    cudaGetDevice(&dev);
    for (int k = 0; k <= (int)root->peers.size(); k++)
        if (cudaSetDevice(context_of(root, k)->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) cudaGetLastError();
    cudaSetDevice(dev);
    host_unregister_all(root);
    return cudaMemcpyAsync(dst, src, bytes, kind, st);
}

// ---- planner ------------------------------------------------------------------------------------------------
static EpiParams make_epi(const tb200_layer_desc& L, const tb200_tensor_desc& tin, const tb200_tensor_desc& tout, bool fc)
{
    EpiParams e{};
    e.in_scale = tin.scale, e.out_scale = tout.scale;
    e.in_zero = tin.zero_point, e.out_zero = tout.zero_point, e.w_zero = L.weight_zero;
    e.activation = L.activation, e.recipe = L.recipe;
    e.is_uint8 = tin.data_type == TB200_DT_UINT8;
    e.fc_rounding = fc ? 1 : 0;
    e.has_bias = L.bias != nullptr;
    e.in_w_scale = e.is_uint8 ? tin.scale * L.weight_scales[0] : 0.f; // fp32 product, as bias_scale in conv_kernel_x86.c:1723
    e.bias_scale = (fc && e.is_uint8 && L.bias_scale != 0.f) ? L.bias_scale : e.in_w_scale; // fc_ref.c:141-146
    // fast-path constants (common.cuh requant_fast): clamps of t = f / s_out with activation and saturation folded in
    const float so = tout.scale;
    const float inf = __builtin_inff();
    const int act = fc ? -1 : L.activation;
    float flo = -inf, fhi = inf; // activation clamp in real units
    if (L.recipe == TB200_RECIPE_HCL || fc)
    {
        if (act == 0) flo = 0.f;
        if (act > 0) flo = 0.f, fhi = 6.f;
    }
    else if (act >= 0)
    {
        if (act == 1) flo = -1.f, fhi = 1.f;
        else flo = 0.f, fhi = (act == 6) ? 6.f : inf;
    }
    e.fast_flo = flo, e.fast_fhi = fhi;
    if (e.is_uint8)
    {
        e.fast_lo = (float)(0 - tout.zero_point), e.fast_hi = (float)(255 - tout.zero_point);
        e.fast_r = 1.0f / so;
        // integer-domain clip + zero point + saturation (common.cuh requant_fast8_i8, the int8 form the uint8 tensor-core epilogues
        // use): the activation bounds become the integers the reference's own division and round() give for them;
        // q' = max(min(q + zp - L, H - L), 0), byte = q' + L
        int q_lo = -30000, q_hi = 30000;
        if (flo > -inf) q_lo = (int)roundf(flo / so);
        if (fhi < inf) q_hi = (int)roundf(fhi / so);
        int Lb = q_lo + tout.zero_point, Hb = q_hi + tout.zero_point;
        Lb = Lb < 0 ? 0 : (Lb > 255 ? 255 : Lb), Hb = Hb > 255 ? 255 : (Hb < 0 ? 0 : Hb);
        const uint32_t add = (uint32_t)(tout.zero_point - Lb) & 0xffffu, mx = (uint32_t)(Hb - Lb) & 0xffffu;
        e.q_add2 = add | (add << 16), e.q_max2 = mx | (mx << 16);
        e.q_byte_add = ((uint32_t)Lb & 0xffu) * 0x01010101u;
    }
    else
    {
        e.fast_lo = -127.f, e.fast_hi = 127.f;
        if (flo > -inf) e.fast_lo = fmaxf(-127.f, flo / so); // fl(x / s_out): the same rounded quotient the reference forms
        if (fhi < inf) e.fast_hi = fminf(127.f, fhi / so);
        e.fast_r = 0.f;
        // integer-domain clamp (common.cuh requant_fast4_i8): [q_lo, q_hi] = what the reference's roundf gives for the
        // clipped bounds; q' = max(min(q - q_lo, q_hi - q_lo), 0), bytes = q' + q_lo
        const int q_lo = (int)roundf(e.fast_lo), q_hi = (int)roundf(e.fast_hi);
        const uint32_t add = (uint32_t)(-q_lo) & 0xffffu, mx = (uint32_t)(q_hi - q_lo) & 0xffffu;
        e.q_add2 = add | (add << 16), e.q_max2 = mx | (mx << 16);
        e.q_byte_add = ((uint32_t)q_lo & 0xffu) * 0x01010101u;
    }
    e.fast_ok = (so > 1e-30f && so < 1e30f && tin.scale > 1e-30f && tin.scale < 1e30f) ? 1 : 0;
    return e;
}

// bytes of the packed B operand of the tensor-core paths: [n_tiles][block_n][K]
static size_t gemm_weight_bytes(int ocp, int k)
{
    const int bn = gemm_block_n(ocp), nt = (ocp + bn - 1) / bn;
    return (size_t)nt * bn * k;
}

static int run_step(tb200_graph* g, const Step& s, cudaStream_t st)
{
    cudaError_t err = cudaSuccess;
    switch (s.kind)
    {
    case K_NCHW2NHWC: err = launch_nchw_to_nhwc(s.in, s.out, s.n, s.c, s.h, s.w_, st); break;
    case K_NHWC2NCHW: err = launch_nhwc_to_nchw(s.in, s.out, s.n, s.c, s.h, s.w_, st); break;
    case K_CONV_STEM: err = launch_conv_stem(s.in, s.w, s.out, s.cs, s.epi, st); break;
    case K_GATHER_TC:
        err = s.wp.valid ? launch_conv_window(s.wp, s.w, s.out, s.cs, s.epi, g->ctx->num_sms, st)
                         : launch_conv_gather_tc(s.in, s.w, s.out, s.cs, s.epi, s.nhwc16, g->ctx->num_sms, st);
        break;
    case K_CONV_DW:
        err = s.dwp.valid ? launch_conv_dw_tma(s.dwp, s.w, s.out, s.cs, s.epi, st) : launch_conv_dw(s.in, s.w, s.out, s.cs, s.epi, st);
        break;
    case K_CONV_DIRECT: err = launch_conv_direct(s.in, s.w, s.out, s.cs, s.epi, st); break;
    case K_GEMM:
    case K_IGEMM: err = launch_gemm_i8(s.gemm, s.epi, s.btab, g->ctx->num_sms, st); break;
    case K_POOL: err = launch_pool(s.in, s.out, s.ps, s.u8, st); break;
    case K_POINTWISE: err = launch_pointwise(s.in, s.in2, s.out, s.bytes, s.pp, s.u8, st); break;
    case K_CONCAT_PART:
        if (s.scale == 1) // 16-channel-aligned input: vectorised, requantisation as a byte table (s.w; nullptr = equal quantisation)
        {
            err = launch_concat_lut(s.in, s.out, (const uint8_t*)s.w, s.npix, s.c, s.c_write, s.cp_in, s.cp_out, s.c_off, st);
            break;
        }
        err = launch_concat_part(s.in, s.out, s.npix, s.c, s.c_write, s.cp_in, s.cp_out, s.c_off, s.s_in, s.z_in, s.s_out, s.z_out, s.u8, st);
        break;
    case K_LUT: err = launch_byte_lut(s.in, s.out, (const uint8_t*)s.w, s.bytes, s.c, s.cp_in, st); break;
    case K_SOFTMAX: err = launch_softmax(s.in, s.out, s.npix, s.c, s.cp_in, s.s_in, s.z_in, s.s_out, s.z_out, s.u8, st); break;
    case K_RESHAPE:
        err = launch_nhwc_to_nchw(s.in, s.scratch, s.n, s.c, s.h, s.w_, st);
        if (err == cudaSuccess) err = launch_nchw_to_nhwc(s.scratch, s.out, s.n, s.oc_, s.oh_, s.ow_, st);
        break;
    case K_UPSAMPLE: err = launch_upsample(s.in, s.out, s.n, s.h, s.w_, s.cp_in, s.scale, st); break;
    case K_COPY: err = cudaMemcpyAsync(s.out, s.in, (size_t)s.bytes, cudaMemcpyDeviceToDevice, st); break;
    }
    if (err != cudaSuccess) return fail(TB200_ERR_CUDA, "launch of %s (layer %d) failed: %s", kStepName[s.kind], s.layer, cudaGetErrorString(err));
    return 0;
}

// the CUDA graphs of `bp` (on the current device) and its steps; bp is then empty
static void destroy_batch_plan(BatchPlan& bp)
{
    for (auto e : bp.cu_execs) if (e) cudaGraphExecDestroy(e);
    for (auto c : bp.cu_graphs) if (c) cudaGraphDestroy(c);
    bp = BatchPlan();
}

static void destroy_graph(tb200_graph* g)
{
    if (!g) return;
    for (tb200_graph* sh : g->shards) destroy_graph(sh);
    g->shards.clear();
    cudaSetDevice(g->ctx->device);
    destroy_batch_plan(g->prepared);
    destroy_batch_plan(g->other);
    for (auto e : g->ev_in) cudaEventDestroy(e);
    for (auto e : g->ev_out) cudaEventDestroy(e);
    if (g->ev_done) cudaEventDestroy(g->ev_done);
    if (g->copy_stream) cudaStreamDestroy(g->copy_stream);
    if (g->d2h_stream) cudaStreamDestroy(g->d2h_stream);
    for (auto p : g->in_nchw_dev) cudaFree(p);
    for (auto p : g->out_nchw_dev) cudaFree(p);
    cudaFree(g->act_arena);
    cudaFree(g->w_arena);
    cudaFree(g->img_stage);
    cudaFree(g->img_desc);
    cudaFreeHost(g->img_desc_host);
    if (g->img_ev) cudaEventDestroy(g->img_ev);
    delete g;
}

// Host-side tables of the unary byte ops (sigmoid, hardswish): inputs are bytes, so the op IS a 256-entry table, computed here
// once per layer with the reference's own C arithmetic (libm exp in double, C round()) -- the device then only permutes bytes,
// bit-exact by construction.  sigmoid/sigmoid_ref.c:84-127 (int8), :129-172 (uint8); hardswish/hardswish_kernel_ref_uint8.c:41-80.
static void build_byte_lut(int op, bool u8, const tb200_tensor_desc& tin, const tb200_tensor_desc& tout, uint8_t* lut)
{
    for (int b = 0; b < 256; b++)
    {
        const float q = u8 ? (float)b : (float)(int)(int8_t)b;
        volatile float x = (q - (float)tin.zero_point) * tin.scale;
        volatile float y;
        if (op == TB200_OP_SIGMOID)
        {
            float t = (x > -30.0f) ? x : -30.0f; // the reference's MIN(x, 30) is overwritten by its MAX(x, -30) (sigmoid_ref.c:110-111)
            y = (float)(1 / (1 + exp((double)-t)));
        }
        else
        {
            volatile float tmp = x + 3.f;
            if (tmp < 0.f) tmp = 0.f;
            if (tmp > 6.f) tmp = 6.f;
            volatile float r = tmp / 6.f;
            y = x * r;
        }
        volatile float z = y / tout.scale;
        volatile float zz = z + (float)tout.zero_point;
        int v = (int)round((double)zz);
        if (u8) v = v > 255 ? 255 : (v < 0 ? 0 : v);
        else v = v > 127 ? 127 : (v < -127 ? -127 : v);
        lut[b] = (uint8_t)(v & 0xff);
    }
}

// Eltwise (SUM / PROD) of two bytes with the arithmetic of eltwise/eltwise_ref.c:311-583 (uint8), 585-845 (int8) -- the statements of
// kernels_direct.cu pointwise_exact_byte -- for tables of node pairs whose two operands are functions of the same byte.
static uint8_t eltwise_byte(bool u8, int elt_type, int a, const tb200_tensor_desc& ta, int b, const tb200_tensor_desc& tb, const tb200_tensor_desc& to)
{
    volatile float f0, f1;
    if (u8) f0 = (float)(a - ta.zero_point) * ta.scale, f1 = (float)(b - tb.zero_point) * tb.scale;
    else f0 = (float)(int)(int8_t)a * ta.scale, f1 = (float)(int)(int8_t)b * tb.scale;
    volatile float f = (elt_type == TB200_ELT_SUM) ? f0 + f1 : f0 * f1;
    volatile float t = f / to.scale;
    int q = (int)roundf(t);
    if (u8)
    {
        q += to.zero_point;
        q = q > 255 ? 255 : (q < 0 ? 0 : q);
    }
    else
        q = q > 127 ? 127 : (q < -127 ? -127 : q);
    return (uint8_t)(q & 0xff);
}

// (leaky) ReLU as a byte table, with the arithmetic of relu/relu_kernel_ref_int8.c:41-94 and relu_kernel_ref_uint8.c:41-96 (the same
// statements as kernels_direct.cu pointwise_exact_byte): used where the node is folded into the max pooling that follows it.
static void build_relu_lut(bool u8, const tb200_tensor_desc& tin, const tb200_tensor_desc& tout, float slope, uint8_t* lut)
{
    for (int b = 0; b < 256; b++)
    {
        volatile float f0 = u8 ? (float)(b - tin.zero_point) * tin.scale : (float)(int)(int8_t)b * tin.scale;
        volatile float f = (f0 < 0.f) ? ((slope == 0.f) ? 0.f : f0 * slope) : f0;
        int q;
        if (u8)
        {
            volatile float t = f / tout.scale;
            volatile float tz = t + (float)tout.zero_point; // relu_kernel_ref_uint8.c:85: the zero point is added inside round()
            q = (int)roundf(tz);
            q = q > 255 ? 255 : (q < 0 ? 0 : q);
        }
        else
        {
            volatile float t = f / tout.scale;
            q = (int)roundf(t);
            q = q > 127 ? 127 : (q < -127 ? -127 : q);
        }
        lut[b] = (uint8_t)(q & 0xff);
    }
}

// ---- graph prerun: planning passes -----------------------------------------------------------------------------
// prerun_one runs them in order; each pass reads the layer plans the earlier ones filled in.

// ---- node fusion (SURVEY.md 8(f)-1), decided from the descriptors alone ----
// [tensor] the one layer that reads it, or -1 when it has no reader, several, or is a graph output: a node may be folded into
// the sole reader of its output
static std::vector<int> sole_readers(const tb200_layer_desc* ls, int num_layers, int num_tensors, const int32_t* output_ids, int num_outputs)
{
    std::vector<int> count(num_tensors, 0), reader(num_tensors, -1);
    for (int li = 0; li < num_layers; li++)
        for (int k = 0; k < ls[li].num_inputs && k < 4; k++)
            if (ls[li].inputs[k] >= 0 && ls[li].inputs[k] < num_tensors) count[ls[li].inputs[k]]++, reader[ls[li].inputs[k]] = li;
    for (int t = 0; t < num_tensors; t++)
        if (count[t] != 1) reader[t] = -1;
    for (int i = 0; i < num_outputs; i++)
        if (output_ids[i] >= 0 && output_ids[i] < num_tensors) reader[output_ids[i]] = -1;
    return reader;
}

// Folds node pairs into one step: `fused` starts as the caller's descriptors and is rewritten in place (folded nodes become
// TB200_OP_NOP_); the links go into the plans.  Not under TB200_PRERUN_NO_GRAPH, whose contract is that every intermediate
// stays readable.
static void fuse_nodes(const tb200_layer_desc* layers, const tb200_tensor_desc* tensors, int num_tensors, const int32_t* output_ids, int num_outputs,
                       std::vector<tb200_layer_desc>& fused, std::vector<LayerPlan>& plan)
{
    const int num_layers = (int)fused.size();
    auto reader_of = [&](const std::vector<int>& sole, int t) { return t >= 0 && t < num_tensors ? sole[t] : -1; };
    // Eltwise -> ReLU where the ReLU's output has its input's quantisation (what the reference's quantisation tool writes,
    // quant_save_graph.cpp:136-200) and the eltwise result has no other reader: the ReLU is then max(byte, zero point) on the
    // requantised bytes (relu_same_scale_kernel), applied inside the eltwise kernel -- one pass over memory instead of two, the
    // intermediate tensor is never stored.
    std::vector<int> sole = sole_readers(layers, num_layers, num_tensors, output_ids, num_outputs);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& E = layers[li];
        const int lj = reader_of(sole, E.output);
        if (E.op != TB200_OP_ELTWISE || lj <= li) continue;
        const tb200_layer_desc& R = layers[lj];
        if (R.op != TB200_OP_RELU || R.negative_slope != 0.f || R.output < 0 || R.output >= num_tensors) continue;
        const tb200_tensor_desc &ti = tensors[E.output], &to = tensors[R.output];
        if (ti.scale != to.scale || ti.zero_point != to.zero_point || ti.data_type != to.data_type) continue;
        if (ti.data_type == TB200_DT_UINT8 && (ti.dims[1] % 16)) continue; // pad lanes of uint8 tensors must stay 0, not the zero point
        bool same = true;
        for (int k = 0; k < 4; k++) same &= ti.dims[k] == to.dims[k];
        if (!same) continue;
        fused[li].output = R.output, plan[li].post_relu = 1;
        fused[lj].op = TB200_OP_NOP_, fused[lj].num_inputs = 0;
    }
    // (Leaky) ReLU -> max pooling whose output keeps the ReLU's quantisation, the ReLU result having no other reader: the ReLU is
    // a non-decreasing byte table, so max(table(x)) == table(max(x)); the pooling reads the convolution's bytes and applies the
    // table to each window's maximum.  One pass over the big tensor disappears.
    sole = sole_readers(fused.data(), num_layers, num_tensors, output_ids, num_outputs);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& R = fused[li];
        const int lj = reader_of(sole, R.output);
        if (R.op != TB200_OP_RELU || lj <= li) continue;
        if (!(R.negative_slope >= 0.f && R.negative_slope <= 1.f)) continue; // the table must be non-decreasing
        const tb200_layer_desc& P = fused[lj];
        if (P.op != TB200_OP_POOL || P.pool_method != TB200_POOL_MAX || P.output < 0 || P.output >= num_tensors) continue;
        const tb200_tensor_desc &tr = tensors[R.output], &tp = tensors[P.output];
        if (tr.scale != tp.scale || tr.zero_point != tp.zero_point || tr.data_type != tp.data_type) continue;
        plan[lj].pool_relu = li;
        fused[lj].inputs[0] = R.inputs[0]; // the pooling reads what the ReLU read
        fused[li].op = TB200_OP_NOP_, fused[li].num_inputs = 0;
    }
    // Sigmoid -> Eltwise-PROD with the Sigmoid's own input (x * sigmoid(x): how an int8 YOLOv5s spells SiLU, SURVEY.md 8(a)): both
    // operands of the product are functions of the same byte of x, so the PAIR is one byte table -- sigmoid's table composed with
    // the reference's eltwise arithmetic, built at prerun -- and one pass (1 read, 1 write) replaces two (3 reads, 2 writes).
    sole = sole_readers(fused.data(), num_layers, num_tensors, output_ids, num_outputs);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& S = fused[li];
        const int lj = reader_of(sole, S.output);
        if (S.op != TB200_OP_SIGMOID || lj <= li) continue;
        const tb200_layer_desc& E = fused[lj];
        if (E.op != TB200_OP_ELTWISE || E.elt_type != TB200_ELT_PROD || E.num_inputs != 2 || plan[lj].post_relu) continue;
        const int other = E.inputs[0] == S.output ? E.inputs[1] : (E.inputs[1] == S.output ? E.inputs[0] : -1);
        if (other != S.inputs[0]) continue;
        plan[lj].silu_sig = li, plan[lj].silu_operand = (E.inputs[0] == S.output) ? 0 : 1;
        fused[lj].op = TB200_OP_LUT2_, fused[lj].num_inputs = 1, fused[lj].inputs[0] = S.inputs[0];
        // E is fused[lj], so this compares the rewritten inputs[0]; nothing reads this axis but the pack-cache key
        fused[lj].axis = (E.inputs[0] == S.output) ? 0 : 1;
        fused[li].op = TB200_OP_NOP_, fused[li].num_inputs = 0;
    }
}

// ---- tensors ----
static int setup_tensors(tb200_graph* g, const tb200_tensor_desc* tensors, int num_tensors, const int32_t* input_ids, int num_inputs, const int32_t* output_ids,
                         int num_outputs)
{
    g->tensors.resize(num_tensors);
    for (int i = 0; i < num_tensors; i++)
    {
        TensorInfo& t = g->tensors[i];
        t.d = tensors[i];
        if (t.d.data_type != TB200_DT_INT8 && t.d.data_type != TB200_DT_UINT8)
            return fail(TB200_ERR_UNSUPPORTED, "tensor %d: data type %d not supported by the H100 backend", i, t.d.data_type);
        for (int k = 0; k < 4; k++)
            if (t.d.dims[k] <= 0) return fail(TB200_ERR_INVALID, "tensor %d: dim %d is %d", i, k, t.d.dims[k]);
        t.cp = cpad(t.d.dims[1]);
        t.nhwc_bytes = (size_t)t.d.dims[0] * t.d.dims[2] * t.d.dims[3] * t.cp;
        t.nchw_bytes = (size_t)t.d.dims[0] * t.d.dims[1] * t.d.dims[2] * t.d.dims[3];
        t.off = 0;
        t.slot_bytes = align_up(t.nhwc_bytes, 1024);
    }
    for (int i = 0; i < num_inputs; i++)
    {
        if (input_ids[i] < 0 || input_ids[i] >= num_tensors) return fail(TB200_ERR_INVALID, "input id out of range");
        g->tensors[input_ids[i]].input_index = i;
        g->input_ids.push_back(input_ids[i]);
    }
    for (int i = 0; i < num_outputs; i++)
    {
        if (output_ids[i] < 0 || output_ids[i] >= num_tensors) return fail(TB200_ERR_INVALID, "output id out of range");
        g->tensors[output_ids[i]].output_index = i;
        g->output_ids.push_back(output_ids[i]);
    }
    return 0;
}

// ---- validation and kernel choice ----
// The kernel of a convolution and the bytes of its packed weights: each kind's predicate next to its weight size.
static int plan_conv(int li, const tb200_layer_desc& L, const TensorInfo& tin, const TensorInfo& tout, bool no_tc, LayerPlan& P)
{
    const int C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3], OC = tout.d.dims[1];
    if (!L.weight || !L.weight_scales) return fail(TB200_ERR_INVALID, "layer %d: conv without weight/scales", li);
    if (L.group < 1 || C % L.group || OC % L.group) return fail(TB200_ERR_INVALID, "layer %d: bad group %d", li, L.group);
    const int oh = (H + L.pad_h0 + L.pad_h1 - (L.dilation_h * (L.kernel_h - 1) + 1)) / L.stride_h + 1;
    const int ow = (W + L.pad_w0 + L.pad_w1 - (L.dilation_w * (L.kernel_w - 1) + 1)) / L.stride_w + 1;
    if (oh != tout.d.dims[2] || ow != tout.d.dims[3] || tout.d.dims[0] != tin.d.dims[0])
        return fail(TB200_ERR_INVALID, "layer %d: conv output shape %dx%d does not match descriptor %dx%d", li, oh, ow, tout.d.dims[2], tout.d.dims[3]);
    const int cg = C / L.group;
    const bool nchw_input = tin.input_index >= 0 && C <= 3; // an RGB / grey stem over the NCHW graph input
    const bool tc = !no_tc && L.group == 1;                                                       // a tensor-core kernel may take it
    const bool plain = L.dilation_h == 1 && L.dilation_w == 1 && L.stride_h == L.stride_w;         // no dilation, one stride
    const bool k3 = L.kernel_h == 3 && L.kernel_w == 3;
    const bool gather = tc && plain && tout.cp <= 256;
    size_t& wsize = P.blob.w_size;
    if (nchw_input && gather && L.kernel_h == L.kernel_w && (L.kernel_h == 3 || L.kernel_h == 7))
        // 3x3 and 7x7 (ResNet) stems: K = C*KH*KW padded to 32*ks (one k-step for a 3x3 stem); uint8 taps outside the image = zero point
        P.kind = K_GATHER_TC, P.reads_nchw = true, wsize = (size_t)tout.cp * 32 * ((C * L.kernel_h * L.kernel_w + 31) / 32);
    else if (tin.input_index >= 0 && C <= 4 && L.group == 1)
        P.kind = K_CONV_STEM, P.reads_nchw = true, wsize = (size_t)tout.cp * L.kernel_h * L.kernel_w * 4;
    else if (gather && k3 && tin.cp == 16)
        P.kind = K_GATHER_TC, P.nhwc16 = 1, wsize = (size_t)tout.cp * 160; // 16-channel input: nine 16-byte taps per pixel, five k-steps
    else if (gather && k3 && tin.cp == 32 && (L.stride_h == 1 || L.stride_h == 2) && window_nhwc_fits(32, tout.cp, L.stride_h))
        P.kind = K_GATHER_TC, P.nhwc16 = 1, wsize = (size_t)tout.cp * 288; // 32-channel input through the window kernel: nine 32-byte taps = nine k-steps
    else if (L.group == C && OC == C && C > 1)
        P.kind = K_CONV_DW, wsize = (size_t)L.kernel_h * L.kernel_w * tin.cp;
    else if (tc && L.kernel_h == 1 && L.kernel_w == 1 && L.stride_h == 1 && L.stride_w == 1 && !L.pad_h0 && !L.pad_h1 && !L.pad_w0 && !L.pad_w1)
        P.kind = K_GEMM, wsize = gemm_weight_bytes(tout.cp, tin.cp);
    else if (tc && plain && (L.stride_h == 1 || L.stride_h == 2) && (L.kernel_h * L.kernel_w == 1 || tin.cp % 32 == 0) &&
             tout.d.dims[3] <= 4096 && L.kernel_h * L.kernel_w <= 64)
        P.kind = K_IGEMM, wsize = gemm_weight_bytes(tout.cp, L.kernel_h * L.kernel_w * tin.cp);
    else
    {
        if (L.group > 1 && ((cg % 4) || ((OC / L.group) % 4)))
            return fail(TB200_ERR_UNSUPPORTED, "layer %d: grouped conv needs channels per group %% 4 == 0", li);
        P.kind = K_CONV_DIRECT;
        wsize = (size_t)tout.cp * L.kernel_h * L.kernel_w * (L.group == 1 ? tin.cp : cg);
    }
    return 0;
}

// Validates every layer, chooses its kernel and lays out the weight arena (g->w_bytes).
static int plan_kernels(tb200_graph* g, std::vector<LayerPlan>& plan)
{
    const int num_layers = (int)g->layers.size(), num_tensors = (int)g->tensors.size();
    const bool no_tc = (g->flags & TB200_PRERUN_NO_TENSORCORE) != 0;
    size_t wtotal = 0;
    auto take = [&](size_t bytes, size_t align) { const size_t off = wtotal; wtotal += align_up(bytes, align); return off; }; // weight arena
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        LayerPlan& P = plan[li];
        if (L.op == TB200_OP_NOP_) continue; // P.kind stays K_NONE
        if (L.num_inputs < 1 || L.num_inputs > 4) return fail(TB200_ERR_INVALID, "layer %d: num_inputs %d", li, L.num_inputs);
        for (int k = 0; k < L.num_inputs; k++)
            if (L.inputs[k] < 0 || L.inputs[k] >= num_tensors) return fail(TB200_ERR_INVALID, "layer %d: input id", li);
        if (L.output < 0 || L.output >= num_tensors) return fail(TB200_ERR_INVALID, "layer %d: output id", li);
        TensorInfo& tin = g->tensors[L.inputs[0]];
        TensorInfo& tout = g->tensors[L.output];
        tout.producer = li;
        if (tin.d.data_type != tout.d.data_type) return fail(TB200_ERR_UNSUPPORTED, "layer %d: mixed data types", li);
        const bool u8 = tin.d.data_type == TB200_DT_UINT8;
        const int C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3];
        if (L.op == TB200_OP_CONV)
        {
            if (const int rc = plan_conv(li, L, tin, tout, no_tc, P)) return rc;
        }
        else if (L.op == TB200_OP_FC)
        {
            if (!L.weight || !L.weight_scales) return fail(TB200_ERR_INVALID, "layer %d: fc without weight/scales", li);
            if (no_tc)
                P.kind = K_CONV_DIRECT, P.blob.w_size = (size_t)tout.cp * H * W * tin.cp; // FC == conv with kernel HxW over the whole input
            else
                P.kind = K_GEMM, P.blob.w_size = gemm_weight_bytes(tout.cp, H * W * tin.cp);
        }
        else if (L.op == TB200_OP_POOL)
            P.kind = K_POOL;
        else if (L.op == TB200_OP_RELU)
            P.kind = K_POINTWISE;
        else if (L.op == TB200_OP_ELTWISE)
        {
            if (L.num_inputs != 2 || (L.elt_type != TB200_ELT_SUM && L.elt_type != TB200_ELT_PROD))
                return fail(TB200_ERR_UNSUPPORTED, "layer %d: eltwise type %d / %d inputs", li, L.elt_type, L.num_inputs);
            P.kind = K_POINTWISE;
        }
        else if (L.op == TB200_OP_CONCAT)
        {
            if (L.axis != 1) return fail(TB200_ERR_UNSUPPORTED, "layer %d: concat axis %d", li, L.axis);
            P.kind = (L.num_inputs == 1) ? K_COPY : K_CONCAT_PART; // concat_kernel_ref_int8.c:45-56: one input is a plain copy
        }
        else if (L.op == TB200_OP_UPSAMPLE)
            P.kind = K_UPSAMPLE;
        else if (L.op == TB200_OP_IDENTITY)
            P.kind = K_COPY;
        else if (L.op == TB200_OP_LUT2_)
            P.kind = K_LUT;
        else if (L.op == TB200_OP_SIGMOID || L.op == TB200_OP_HARDSWISH)
        {
            // the reference has no int8 hardswish (hardswish_ref.c:59-66): nothing to be identical to
            if (L.op == TB200_OP_HARDSWISH && !u8) return fail(TB200_ERR_UNSUPPORTED, "layer %d: int8 hardswish has no reference kernel", li);
            P.kind = K_LUT;
        }
        else if (L.op == TB200_OP_SOFTMAX)
        {
            if (L.axis != 1) return fail(TB200_ERR_UNSUPPORTED, "layer %d: softmax axis %d (only the channel axis)", li, L.axis);
            P.kind = K_SOFTMAX;
        }
        else if (L.op == TB200_OP_RESHAPE)
        {
            if (tin.nchw_bytes != tout.nchw_bytes || tin.d.dims[0] != tout.d.dims[0])
                return fail(TB200_ERR_INVALID, "layer %d: reshape changes the element count or the batch", li);
            // NHWC(pad) == NCHW order when the tensor is a vector per image or has one channel: a plain copy then
            const bool same = (H * W == 1 && tout.d.dims[2] * tout.d.dims[3] == 1) || (C == tout.d.dims[1] && H == tout.d.dims[2] && W == tout.d.dims[3]);
            P.kind = same ? K_COPY : K_RESHAPE;
        }
        else
            return fail(TB200_ERR_UNSUPPORTED, "layer %d: op %d", li, L.op);

        if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
        {
            P.k = L.op == TB200_OP_FC ? (size_t)C * H * W : (size_t)(C / L.group) * L.kernel_h * L.kernel_w;
            P.u8_tc = u8 && (P.kind == K_GEMM || P.kind == K_IGEMM || P.kind == K_GATHER_TC);
            P.gemm_zp = u8 ? 1 + L.weight_zero : 0;
            P.blob.w_off = take(P.blob.w_size, 1024);
            P.blob.bias_off = take((size_t)tout.cp * 4, 256);
            P.blob.scale_off = take((size_t)tout.cp * 4, 256);
            P.blob.fast_off = take((size_t)tout.cp * 8, 256);
            // [border patterns][OCp] int32, see pack_border_table
            const size_t patterns = (u8 && P.kind == K_IGEMM) ? (size_t)(L.pad_h0 + 1) * (L.kernel_h + 1) * (L.pad_w0 + 1) * (L.kernel_w + 1) : 0;
            P.blob.btab_off = take(patterns * tout.cp * 4, 256);
        }
        if (P.kind == K_LUT || (P.kind == K_POOL && P.pool_relu >= 0))
            P.blob.w_off = take(256, 1); // 256-byte table; part of the arena so that it travels with the single broadcast
        if (P.kind == K_CONCAT_PART) P.blob.w_off = take(256 * 4, 1); // one requantisation table per input
        // which graph inputs need an NHWC copy (everything except a stem conv reads NHWC)
        for (int k = 0; k < L.num_inputs; k++)
            if (g->tensors[L.inputs[k]].input_index >= 0 && !P.reads_nchw) g->tensors[L.inputs[k]].nhwc_needed = true;
    }
    for (int id : g->output_ids)
        if (g->tensors[id].input_index >= 0) g->tensors[id].nhwc_needed = true;
    g->w_bytes = wtotal ? wtotal : 1024;
    return 0;
}

// ---- activation arena: one 1 KiB-aligned slot per tensor; a slot is handed on once the tensor's last consumer has run
//      (first-fit over a coalescing free list, the role of source/device/cpu/cpu_pool.c:253-439).  Graph inputs and outputs
//      keep their slots; with TB200_PRERUN_NO_GRAPH (debug: every intermediate stays readable) nothing is reused. ----
static void plan_activation_arena(tb200_graph* g, std::vector<LayerPlan>& plan)
{
    const int num_layers = (int)g->layers.size(), num_tensors = (int)g->tensors.size();
    const bool reuse = !(g->flags & TB200_PRERUN_NO_GRAPH);
    for (int li = 0; li < num_layers; li++)
        for (int k = 0; k < g->layers[li].num_inputs; k++) g->tensors[g->layers[li].inputs[k]].last_use = li;
    struct Blk { size_t off, bytes; };
    std::vector<Blk> free_list; // sorted by offset
    size_t top = 0;
    auto alloc = [&](size_t bytes) -> size_t
    {
        for (size_t i = 0; i < free_list.size(); i++)
            if (free_list[i].bytes >= bytes)
            {
                const size_t off = free_list[i].off;
                free_list[i].off += bytes, free_list[i].bytes -= bytes;
                if (!free_list[i].bytes) free_list.erase(free_list.begin() + i);
                return off;
            }
        if (!free_list.empty() && free_list.back().off + free_list.back().bytes == top)
        {
            // grow the trailing free block instead of leaving it stranded
            const size_t off = free_list.back().off;
            top = off + bytes;
            free_list.pop_back();
            return off;
        }
        const size_t off = top;
        top += bytes;
        return off;
    };
    auto release = [&](size_t off, size_t bytes)
    {
        if (!reuse || !bytes) return;
        size_t i = 0;
        while (i < free_list.size() && free_list[i].off < off) i++;
        free_list.insert(free_list.begin() + i, Blk{off, bytes});
        if (i + 1 < free_list.size() && free_list[i].off + free_list[i].bytes == free_list[i + 1].off)
            free_list[i].bytes += free_list[i + 1].bytes, free_list.erase(free_list.begin() + i + 1);
        if (i > 0 && free_list[i - 1].off + free_list[i - 1].bytes == free_list[i].off)
            free_list[i - 1].bytes += free_list[i].bytes, free_list.erase(free_list.begin() + i);
    };
    std::vector<char> placed(num_tensors, 0), freed(num_tensors, 0);
    for (int i = 0; i < num_tensors; i++)
    {
        TensorInfo& t = g->tensors[i];
        g->act_unshared_bytes += t.slot_bytes;
        if (t.producer < 0 && t.last_use < 0 && t.input_index < 0 && t.output_index < 0)
        {
            placed[i] = 1; // neither produced nor read (e.g. the intermediate of a folded node pair): no slot
            g->act_unshared_bytes -= t.slot_bytes;
            continue;
        }
        if (t.producer < 0) t.off = alloc(t.slot_bytes), placed[i] = 1; // graph inputs
    }
    auto permanent = [&](const TensorInfo& t) { return t.input_index >= 0 || t.output_index >= 0 || t.producer < 0; };
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        if (L.op == TB200_OP_NOP_) continue;
        TensorInfo& to = g->tensors[L.output];
        if (!placed[L.output]) to.off = alloc(to.slot_bytes), placed[L.output] = 1;
        if (plan[li].kind == K_RESHAPE)
        {
            const size_t sb = align_up(to.nchw_bytes, 1024);
            plan[li].scratch_off = alloc(sb);
            g->act_unshared_bytes += sb;
            release(plan[li].scratch_off, sb);
        }
        for (int k = 0; k < L.num_inputs; k++)
        {
            const int id = L.inputs[k];
            TensorInfo& ti = g->tensors[id];
            if (ti.last_use == li && !permanent(ti) && !freed[id]) release(ti.off, ti.slot_bytes), freed[id] = 1;
        }
        if (to.last_use < li && !permanent(to) && !freed[L.output]) release(to.off, to.slot_bytes), freed[L.output] = 1; // dead value
    }
    g->act_bytes = top;
}

// The arenas and the NCHW staging buffers of the graph's inputs and outputs.
static int alloc_device_buffers(tb200_graph* g)
{
    const size_t act = g->act_bytes;
    CUDA_OK(cudaMalloc(&g->act_arena, act ? act : 1024));
    // pad lanes of every tensor are (re)written by its producer; the initial fill only matters for debugging reads
    CUDA_OK(cudaMemsetAsync(g->act_arena, (g->flags & TB200_PRERUN_POISON_ARENA) ? 0xA5 : 0, act ? act : 1024, g->ctx->stream));
    for (auto& t : g->tensors) t.dev = g->act_arena + t.off;
    CUDA_OK(cudaMalloc(&g->w_arena, g->w_bytes));
    for (int id : g->input_ids)
    {
        uint8_t* p = nullptr;
        CUDA_OK(cudaMalloc(&p, g->tensors[id].nchw_bytes));
        g->in_nchw_dev.push_back(p);
    }
    for (int id : g->output_ids)
    {
        uint8_t* p = nullptr;
        CUDA_OK(cudaMalloc(&p, g->tensors[id].nchw_bytes));
        g->out_nchw_dev.push_back(p);
    }
    return 0;
}

// ---- the fast-epilogue proofs, per conv / FC layer.  Decided from the descriptors alone so that every rank of a sharded job
//      reaches the same arena format. ----
static void prove_fast_epilogues(const tb200_graph* g, std::vector<LayerPlan>& plan)
{
    for (size_t li = 0; li < g->layers.size(); li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        LayerPlan& P = plan[li];
        if (L.op != TB200_OP_CONV && L.op != TB200_OP_FC) continue;
        const TensorInfo& tin = g->tensors[L.inputs[0]];
        const TensorInfo& tout = g->tensors[L.output];
        const bool u8 = tin.d.data_type == TB200_DT_UINT8;
        const int OC = tout.d.dims[1];
        // may the int8 fast epilogue fold the bias add into its FMA?  (common.cuh requant_fast_bits<.., FUSE>)
        if (L.op == TB200_OP_CONV && !u8)
        {
            bool fuse = true;
            for (int o = 0; o < OC; o++)
            {
                const double bm = (double)(L.bias ? L.bias[o] : 0) * (double)tin.d.scale * (double)L.weight_scales[o] / (double)tout.d.scale;
                if (!(bm >= -100.0 && bm <= 100.0)) fuse = false;
            }
            P.fuse_bias = fuse ? 1 : 0;
        }
        // uint8 tensor-core layers use the int8 form of the fast epilogue: t = fl((float)(acc_true + bias) * M), M = fl(s_in*s_w/s_out).
        // The reference forms f = fl(fl(acc*S) + fl(bias*S)) and t_ref = fl(f / s_out): |t - t_ref| <= 2^-24 (2|bias*M| + 5|t|), which
        // stays inside the 2^-13 tie guard for every in-range t (|t| <= 255) as long as |bias*M| <= 250 -- checked here per channel;
        // an FC whose bias tensor carries its own scale (fc_ref.c:141-146) cannot fold the bias into the integer sum at all.
        // Layers that fail the check take the exact epilogue.
        if (P.u8_tc)
        {
            const float S = tin.d.scale * L.weight_scales[0];
            if (L.op == TB200_OP_FC && L.bias && L.bias_scale != 0.f && L.bias_scale != S) P.fast_ok = false;
            const double M = (double)tin.d.scale * (double)L.weight_scales[0] / (double)tout.d.scale;
            for (int o = 0; o < OC && L.bias; o++)
                if (!(fabs((double)L.bias[o] * M) <= 250.0)) P.fast_ok = false;
        }
        // the int8 fast epilogue rounds BEFORE it clamps (integer-domain clamp on 16-bit lanes, common.cuh): prove from the
        // weights that no reachable accumulator can leave the 16-bit range after scaling, else use the exact path
        for (int o = 0; o < OC; o++)
        {
            double sumabs = 0;
            if (u8)
                for (size_t k = 0; k < P.k; k++) sumabs += abs((int)((const uint8_t*)L.weight)[(size_t)o * P.k + k] - L.weight_zero);
            else
                for (size_t k = 0; k < P.k; k++) sumabs += abs((int)((const int8_t*)L.weight)[(size_t)o * P.k + k]);
            const double M = (double)tin.d.scale * (double)L.weight_scales[u8 ? 0 : o] / (double)tout.d.scale;
            const double bound = ((u8 ? 255.0 : 128.0) * sumabs + fabs((double)(L.bias ? L.bias[o] : 0))) * fabs(M) + 256.0;
            if (!(bound < 32000.0)) P.fast_ok = false;
        }
    }
}

// ---- weight packing: a host image of the arena, one H2D copy ----
// Per-input requantisation of concat_kernel_ref_int8.c:70-80 (roundf(q * (s_in / s_out)), including its clamp of values below
// -127 to +127) and concat_kernel_ref_uint8.c:82 (roundf((q - zp_in) * (s_in / s_out) + zp_out), the zero point inside the
// rounding, clamp) as byte tables, 256 bytes per input.
static void pack_concat_tables(const tb200_graph* g, const tb200_layer_desc& L, uint8_t* dst)
{
    const tb200_tensor_desc& to = g->tensors[L.output].d;
    for (int k = 0; k < L.num_inputs && k < 4; k++)
    {
        const tb200_tensor_desc& ti = g->tensors[L.inputs[k]].d;
        uint8_t* lut = dst + 256 * k;
        for (int b = 0; b < 256; b++)
        {
            int q;
            if (ti.data_type == TB200_DT_UINT8)
            {
                volatile float rs = ti.scale / to.scale;
                volatile float f = (float)(b - ti.zero_point) * rs;
                volatile float t = f + (float)to.zero_point;
                q = (int)roundf(t);
                q = q > 255 ? 255 : (q < 0 ? 0 : q);
            }
            else
            {
                volatile float rs = ti.scale / to.scale;
                volatile float t = (float)(int)(int8_t)b * rs;
                q = (int)roundf(t);
                q = (q > 127 ? 127 : (q < -127 ? 127 : q)) & 0xff; // sic
            }
            lut[b] = (uint8_t)q;
        }
    }
}

// x -> sigmoid(x) (its own requantisation, the Sigmoid node's output tensor) -> eltwise product with x.  L is the fused
// product (it reads x), S the folded Sigmoid, `operand` the product's operand that S was.
static void pack_silu_table(const tb200_graph* g, const tb200_layer_desc& L, const tb200_layer_desc& S, int operand, uint8_t* lut)
{
    const tb200_tensor_desc &tx = g->tensors[L.inputs[0]].d, &ts = g->tensors[S.output].d, &to = g->tensors[L.output].d;
    const bool u8 = tx.data_type == TB200_DT_UINT8;
    uint8_t sig[256];
    build_byte_lut(TB200_OP_SIGMOID, u8, tx, ts, sig);
    for (int b = 0; b < 256; b++)
        lut[b] = (operand == 0) ? eltwise_byte(u8, TB200_ELT_PROD, sig[b], ts, b, tx, to) : eltwise_byte(u8, TB200_ELT_PROD, b, tx, sig[b], ts, to);
}

// The weights of a conv / FC layer in its kernel's layout.
static void pack_conv_weights(const tb200_layer_desc& L, const LayerPlan& P, const TensorInfo& tin, const TensorInfo& tout, uint8_t* dst)
{
    const int C = tin.d.dims[1], OC = tout.d.dims[1], KH = L.kernel_h, KW = L.kernel_w, cg = C / L.group;
    const uint8_t* src = (const uint8_t*)L.weight;
    if (P.kind == K_CONV_DW)
    {
        for (int c = 0; c < C; c++)
            for (int t = 0; t < KH * KW; t++) dst[(size_t)t * tin.cp + c] = src[(size_t)c * KH * KW + t];
        return;
    }
    if (P.kind == K_GATHER_TC && P.nhwc16)
    {
        // 16- / 32-channel NHWC input: k = (kh*3 + kw)*Cp + c; rows of 160 bytes (the last 16 stay 0) / 288 bytes
        const size_t rowb = tin.cp == 16 ? 160 : 288;
        for (int o = 0; o < OC; o++)
            for (int c = 0; c < C; c++)
                for (int t = 0; t < 9; t++) dst[(size_t)o * rowb + t * tin.cp + c] = src[((size_t)o * C + c) * 9 + t];
        return;
    }
    if (P.kind == K_GATHER_TC)
    {
        // [OC][C][KH][KW] is already k = (c*KH + kh)*KW + kw order: one zero-padded row of 32*ks bytes per channel
        const size_t kp = ((P.k + 31) / 32) * 32;
        for (int o = 0; o < OC; o++) memcpy(dst + (size_t)o * kp, src + (size_t)o * P.k, P.k);
        return;
    }
    // One row of `taps` groups of cgp bytes per output channel; an FC is a conv with kernel HxW over the whole input
    // ([OC][C*H*W], the NCHW flatten of fc_ref.c:313-359 -> [row][H][W][Cp]).
    const bool fc = L.op == TB200_OP_FC, gemm = P.kind == K_GEMM || P.kind == K_IGEMM, u8 = tin.d.data_type == TB200_DT_UINT8;
    const int taps = fc ? tin.d.dims[2] * tin.d.dims[3] : KH * KW, cin = fc ? C : cg;
    const int cgp = P.kind == K_CONV_STEM ? 4 : ((fc || L.group == 1) ? tin.cp : cg);
    const size_t krow = (size_t)taps * cgp;
    for (int o = 0; o < OC; o++)
        for (int c = 0; c < cin; c++)
            for (int t = 0; t < taps; t++) dst[((size_t)o * taps + t) * cgp + c] = src[((size_t)o * cin + c) * taps + t];
    if (!(gemm && u8)) return;
    // the tensor cores form sum x*(w - 128): B = w - 128 as int8 (the epilogue adds (128 - zw) * sum(x)), or plain w when
    // zw == 0.  Real K positions only; pad positions stay 0 (x is 0 there anyway).
    if (L.weight_zero != 0)
        for (int o = 0; o < OC; o++)
            for (int t = 0; t < taps; t++)
                for (int c = 0; c < cin; c++)
                {
                    uint8_t& w = dst[(size_t)o * krow + (size_t)t * cgp + c];
                    w = (uint8_t)(int8_t)((int)w - 128);
                }
}

// uint8 K_IGEMM: what the taps that fall into the padding must give back.  A tap t contributes zx*(sum_c w - Cin*zw) when it is
// inside the image.  A pixel whose window is cut by a rows at the top, b at the bottom, c columns on the left and d on the right
// misses the taps {kh < a or kh >= KH-b or kw < c or kw >= KW-d}; the table holds the SUM of their corrections per channel, index
// ((a*(KH+1) + b)*(pw+1) + c)*(KW+1) + d (gemm_tcgen05.cu border_pattern), so a border row costs one vector load per four channels
// instead of a loop over taps.
static void pack_border_table(const tb200_layer_desc& L, const TensorInfo& tin, const TensorInfo& tout, int32_t* pt)
{
    const int C = tin.d.dims[1], OC = tout.d.dims[1], KH = L.kernel_h, KW = L.kernel_w, taps = KH * KW;
    const uint8_t* src = (const uint8_t*)L.weight;
    std::vector<int64_t> tapc((size_t)taps * OC, 0);
    for (int o = 0; o < OC; o++)
        for (int t = 0; t < taps; t++)
        {
            int64_t sw = 0;
            for (int c = 0; c < C; c++) sw += src[((size_t)o * C + c) * taps + t];
            tapc[(size_t)t * OC + o] = (int64_t)tin.d.zero_point * (sw - (int64_t)C * L.weight_zero);
        }
    for (int a = 0; a <= L.pad_h0; a++)
        for (int b2 = 0; b2 <= KH; b2++)
            for (int c2 = 0; c2 <= L.pad_w0; c2++)
                for (int d2 = 0; d2 <= KW; d2++)
                {
                    const size_t pid = (((size_t)a * (KH + 1) + b2) * (L.pad_w0 + 1) + c2) * (KW + 1) + d2;
                    for (int o = 0; o < OC; o++)
                    {
                        int64_t sum = 0;
                        for (int kh = 0; kh < KH; kh++)
                            for (int kw = 0; kw < KW; kw++)
                                if (kh < a || kh >= KH - b2 || kw < c2 || kw >= KW - d2) sum += tapc[(size_t)(kh * KW + kw) * OC + o];
                        pt[pid * tout.cp + o] = (int32_t)sum;
                    }
                }
}

// Bias, weight scales and the fast epilogue's per-channel constants (float2 per channel: multiplier | bias term, bias bits).
static void pack_epilogue_consts(const tb200_layer_desc& L, const LayerPlan& P, const TensorInfo& tin, const TensorInfo& tout, uint8_t* img)
{
    const bool u8 = tin.d.data_type == TB200_DT_UINT8, fc = L.op == TB200_OP_FC;
    const int OC = tout.d.dims[1];
    int32_t* b = (int32_t*)(img + P.blob.bias_off);
    float* sc = (float*)(img + P.blob.scale_off);
    float* fm = (float*)(img + P.blob.fast_off);
    for (int o = 0; o < tout.cp; o++)
    {
        b[o] = (L.bias && o < OC) ? L.bias[o] : 0;
        sc[o] = u8 ? L.weight_scales[0] : (o < OC ? L.weight_scales[o] : 1.f);
        if (P.u8_tc)
        {
            // tensor-core layers: the int8 layout { M[2k], M[2k+1], y[2k], y[2k+1] } with y = corr[oc] + bias[oc] as an integer
            // (corr[oc] = -zx*sum_k w + K*zx*zw: what the zero points contribute when every tap is inside the image)
            float* fmM = fm + (size_t)(o >> 1) * 4 + (o & 1);
            float* fmY = fmM + 2;
            int32_t y = 0;
            if (o < OC)
            {
                int64_t wsum = 0; // the raw weight bytes of channel o
                for (size_t k = 0; k < P.k; k++) wsum += ((const uint8_t*)L.weight)[(size_t)o * P.k + k];
                y = (int32_t)(-(int64_t)tin.d.zero_point * wsum + (int64_t)P.k * tin.d.zero_point * L.weight_zero + (int64_t)b[o]);
            }
            *fmM = (o >= OC) ? 0.f : (float)((double)tin.d.scale * (double)L.weight_scales[0] / (double)tout.d.scale);
            memcpy(fmY, &y, 4);
        }
        else if (u8)
        {
            // the bias term in real units, rounded exactly as the reference rounds it; the .y lane stays 0
            const float S = tin.d.scale * L.weight_scales[0];
            // FC: fc_ref.c:141-146 multiplies by the BIAS TENSOR's own scale (normally s_in*s_w, but the file decides)
            const float Sb = (fc && L.bias_scale != 0.f) ? L.bias_scale : S;
            fm[2 * o] = (o >= OC) ? 0.f : (fc ? (float)b[o] * Sb : ((L.recipe == TB200_RECIPE_HCL) ? (float)b[o] * S : ((float)b[o] * tin.d.scale) * L.weight_scales[0]));
        }
        else
        {
            // channel pairs interleaved (common.cuh FastPar4): { M[2k], M[2k+1], y[2k], y[2k+1] }
            float* fmM = fm + (size_t)(o >> 1) * 4 + (o & 1);
            float* fmY = fmM + 2;
            if (o >= OC) *fmM = 0.f;
            else if (fc) *fmM = (tin.d.scale * sc[o]) / tout.d.scale; // fc_ref.c:225, the reference's own requant scale
            else *fmM = (float)((double)tin.d.scale * (double)sc[o] / (double)tout.d.scale);
            if (P.fuse_bias) *fmY = (o >= OC) ? 0.f : (float)((double)b[o] * (double)*fmM); // fl(bias*M)
            else memcpy(fmY, &b[o], 4);
        }
    }
}

// Every layer's part of the arena image `img` (zero-filled, g->w_bytes).
static void pack_arena_image(const tb200_graph* g, const std::vector<LayerPlan>& plan, uint8_t* img)
{
    for (size_t li = 0; li < g->layers.size(); li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        const LayerPlan& P = plan[li];
        uint8_t* dst = img + P.blob.w_off;
        if (P.kind == K_CONCAT_PART)
            pack_concat_tables(g, L, dst);
        else if (P.kind == K_POOL && P.pool_relu >= 0) // tin = what the folded ReLU read, its own output quantisation = the pooling's
            build_relu_lut(g->tensors[L.inputs[0]].d.data_type == TB200_DT_UINT8, g->tensors[L.inputs[0]].d, g->tensors[L.output].d,
                           g->layers[P.pool_relu].negative_slope, dst);
        else if (P.kind == K_LUT && L.op == TB200_OP_LUT2_)
            pack_silu_table(g, L, g->layers[P.silu_sig], P.silu_operand, dst);
        else if (P.kind == K_LUT)
            build_byte_lut(L.op, g->tensors[L.inputs[0]].d.data_type == TB200_DT_UINT8, g->tensors[L.inputs[0]].d, g->tensors[L.output].d, dst);
        else if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
        {
            const TensorInfo& tin = g->tensors[L.inputs[0]];
            const TensorInfo& tout = g->tensors[L.output];
            pack_conv_weights(L, P, tin, tout, dst);
            if (P.u8_tc && P.kind == K_IGEMM) pack_border_table(L, tin, tout, (int32_t*)(img + P.blob.btab_off));
            pack_epilogue_consts(L, P, tin, tout, img);
        }
    }
}

// TB200_DEBUG_HASH >= 2: the packed constants and hashes of every conv / FC layer's part of the arena image.
static void debug_print_pack(const tb200_graph* g, const std::vector<LayerPlan>& plan, const uint8_t* img)
{
    for (size_t li = 0; li < g->layers.size(); li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        const LayerPlan& P = plan[li];
        if (L.op != TB200_OP_CONV && L.op != TB200_OP_FC) continue;
        const TensorInfo& ti = g->tensors[L.inputs[0]];
        const TensorInfo& to = g->tensors[L.output];
        const size_t ocp = to.cp;
        const float* fmv = (const float*)(img + P.blob.fast_off);
        int y0, y1;
        memcpy(&y0, fmv + 2, 4), memcpy(&y1, fmv + 3, 4);
        fprintf(stderr, "[tb200 dbg] pack layer %zu consts: in(%.9g, %d) out(%.9g, %d) ws %.9g wz %d M %.9g %.9g y %d %d bias0 %d\n", li, ti.d.scale, ti.d.zero_point,
                to.d.scale, to.d.zero_point, L.weight_scales[0], L.weight_zero, fmv[0], fmv[1], y0, y1, L.bias ? L.bias[0] : 0);
        fprintf(stderr, "[tb200 dbg] pack layer %zu kind %d: w %016llx (%zu) bias %016llx scale %016llx fast %016llx fuse %d fast_ok %d\n", li, P.kind,
                (unsigned long long)fnv1a(img + P.blob.w_off, P.blob.w_size), P.blob.w_size, (unsigned long long)fnv1a(img + P.blob.bias_off, ocp * 4),
                (unsigned long long)fnv1a(img + P.blob.scale_off, ocp * 4), (unsigned long long)fnv1a(img + P.blob.fast_off, ocp * 8), P.fuse_bias, (int)P.fast_ok);
    }
}

// ---- packed-weight cache (tb200_pack_cache_dir / TG_B200_PACK_CACHE; SURVEY.md 8(f)-3): the image is keyed by a hash of
//      everything it depends on -- descriptors, kernel choices, weights, biases, scales -- and a second prerun of the same model
//      reads it back instead of packing again (the analogue of keeping conv_hcl_prerun's interleaved weights,
//      conv_kernel_x86.c:2137-2209, next to the tmfile).  What is hashed, and in which order, is part of the cache format. ----
static const uint64_t kPackMagic = 0x3032424b43415054ull + TB200_PACK_FORMAT;

static uint64_t pack_cache_key(const tb200_graph* g, const std::vector<LayerPlan>& plan)
{
    uint64_t h = kFnvBasis;
    auto mix = [&](const void* p, size_t n) { h = fnv1a(p, n, h); };
    const int num_layers = (int)g->layers.size();
    const int ver = TB200_PACK_FORMAT;
    mix(&ver, sizeof ver), mix(&g->w_bytes, sizeof g->w_bytes), mix(&num_layers, sizeof num_layers);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        const LayerPlan& P = plan[li];
        mix(&P.kind, sizeof(int)), mix(&P.blob, sizeof(WeightBlob)), mix(&P.fuse_bias, sizeof(int));
        mix(&L.op, offsetof(tb200_layer_desc, weight)); // every scalar field up to the pointers
        mix(&L.weight_zero, sizeof L.weight_zero), mix(&L.bias_scale, sizeof L.bias_scale);
        for (int k = 0; k < L.num_inputs && k < 4; k++) mix(&g->tensors[L.inputs[k]].d, sizeof(tb200_tensor_desc));
        if (L.op != TB200_OP_NOP_) mix(&g->tensors[L.output].d, sizeof(tb200_tensor_desc));
        if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
        {
            const TensorInfo& ti = g->tensors[L.inputs[0]];
            const int OC = g->tensors[L.output].d.dims[1];
            mix(L.weight, (size_t)OC * P.k);
            if (L.bias) mix(L.bias, (size_t)OC * 4);
            mix(L.weight_scales, ti.d.data_type == TB200_DT_UINT8 ? 4 : (size_t)OC * 4);
        }
    }
    // batch-dependent fields of the tensor descriptors were hashed too: a cache entry is per (model, batch) like a plan
    return h;
}

static bool pack_cache_load(const std::string& path, uint64_t key, std::vector<uint8_t>& img)
{
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    uint64_t hdr[3] = {0, 0, 0};
    const bool hit = fread(hdr, sizeof hdr, 1, f) == 1 && hdr[0] == kPackMagic && hdr[1] == key && hdr[2] == img.size() &&
                     fread(img.data(), 1, img.size(), f) == img.size();
    fclose(f);
    if (!hit) std::fill(img.begin(), img.end(), 0); // a truncated file must not leave bytes that packing does not overwrite
    return hit;
}

// write-then-rename so that a concurrent reader never sees a partial file; failure to write is not an error
static void pack_cache_store(const std::string& path, uint64_t key, const std::vector<uint8_t>& img)
{
    const std::string tmp = path + ".tmp" + std::to_string((long long)getpid());
    if (FILE* f = fopen(tmp.c_str(), "wb"))
    {
        const uint64_t hdr[3] = {kPackMagic, key, img.size()};
        const bool ok = fwrite(hdr, sizeof hdr, 1, f) == 1 && fwrite(img.data(), 1, img.size(), f) == img.size();
        fclose(f);
        if (!ok || rename(tmp.c_str(), path.c_str()) != 0) remove(tmp.c_str());
    }
}

// Fills the weight arena: from the pack cache when it holds this model, else by packing (and then storing it there).
static int upload_weights(tb200_graph* g, const std::vector<LayerPlan>& plan)
{
    std::vector<uint8_t> img(g->w_bytes, 0);
    const std::string dir = pack_cache_dir();
    std::string cache_path;
    uint64_t key = 0;
    bool cache_hit = false;
    if (!dir.empty())
    {
        key = pack_cache_key(g, plan);
        char name[64];
        snprintf(name, sizeof name, "/tb200_%016llx.pack", (unsigned long long)key);
        cache_path = dir + name;
        cache_hit = pack_cache_load(cache_path, key, img);
    }
    g->pack_cache_state = cache_path.empty() ? 0 : (cache_hit ? 2 : 1);
    if (!cache_hit) pack_arena_image(g, plan, img.data());
    if (getenv("TB200_DEBUG_HASH") && atoi(getenv("TB200_DEBUG_HASH")) >= 2) debug_print_pack(g, plan, img.data());
    if (!cache_path.empty() && !cache_hit) pack_cache_store(cache_path, key, img);
    CUDA_OK(host_copy(g->ctx, g->w_arena, img.data(), g->w_bytes, cudaMemcpyHostToDevice, g->ctx->stream));
    CUDA_OK(cudaStreamSynchronize(g->ctx->stream));
    return 0;
}

// ---- pipeline chunks: an even batch of 32 or more is cut into two chunks (images are independent units) so that `run` can
//      overlap the H2D copy of the second with the kernels of the first; each chunk owns a slice of every tensor ----
static void plan_chunks(const tb200_graph* g, int Ntot, BatchPlan& bp)
{
    bool same_batch = true;
    for (auto& t : g->tensors) same_batch &= (t.d.dims[0] == g->tensors[0].d.dims[0]);
    int K = 1;
    std::vector<int> cfirst{0}, ccount{Ntot};
    if (same_batch && !(g->flags & TB200_PRERUN_NO_GRAPH) && Ntot >= 32 && Ntot % 2 == 0)
    {
        K = 2;
        // from 64 images two chunks of 1/4 and 3/4: the kernels only ever wait for the first quarter of the input (measured on
        // MobileNet-v1 b=256 through tb200_graph_run: 1.78 ms vs 1.92 ms for two halves; three-way splits 1.85-1.87 ms)
        const int a = Ntot >= 64 ? ((Ntot / 4 + 7) / 8) * 8 : Ntot / 2;
        cfirst = {0, a}, ccount = {a, Ntot - a};
    }
    bp.chunks = K;
    bp.chunk_first = cfirst, bp.chunk_count = ccount;
    bp.chunk_steps.resize(K > 1 ? K : 0);
}

// ---- step building ----
// Images [first, first + nb) of a batch of ntot: where a tensor's slice starts, and its NHWC bytes.
struct Slice
{
    int first, nb, ntot;
    size_t off(size_t total_bytes) const { return (total_bytes / (size_t)ntot) * (size_t)first; }
    uint8_t* dev(const TensorInfo& t) const { return t.dev + off(t.nhwc_bytes); }
    long long bytes(const TensorInfo& t) const { return (long long)(t.nhwc_bytes / (size_t)ntot * (size_t)nb); }
};

static int fill_conv_step(tb200_graph* g, int li, const LayerPlan& P, const Slice& sl, BatchPlan* work, Step& s)
{
    const tb200_layer_desc& L = g->layers[li];
    const TensorInfo& tin = g->tensors[L.inputs[0]];
    const TensorInfo& tout = g->tensors[L.output];
    const int N = sl.nb, C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3];
    const int OC = tout.d.dims[1], OH = tout.d.dims[2], OW = tout.d.dims[3];
    const bool fc = L.op == TB200_OP_FC;
    s.w = g->w_arena + P.blob.w_off;
    s.epi = make_epi(L, tin.d, tout.d, fc);
    s.epi.bias = (const int32_t*)(g->w_arena + P.blob.bias_off);
    s.epi.w_scale = (const float*)(g->w_arena + P.blob.scale_off);
    s.epi.fast_par = (const float2*)(g->w_arena + P.blob.fast_off);
    s.btab = (const int32_t*)(g->w_arena + P.blob.btab_off);
    s.epi.fuse_bias = P.fuse_bias;
    if (!P.fast_ok) s.epi.fast_ok = 0;
    ConvShape& cs = s.cs;
    cs.n = N, cs.h = H, cs.w = W, cs.c = C, cs.cp = tin.cp, cs.oh = OH, cs.ow = OW, cs.oc = OC, cs.ocp = tout.cp;
    if (fc)
    {
        cs.kh = H, cs.kw = W, cs.sh = cs.sw = 1, cs.ph0 = cs.pw0 = 0, cs.dh = cs.dw = 1, cs.group = 1;
        cs.cg = C, cs.cgp = tin.cp;
    }
    else
    {
        cs.kh = L.kernel_h, cs.kw = L.kernel_w, cs.sh = L.stride_h, cs.sw = L.stride_w, cs.ph0 = L.pad_h0, cs.pw0 = L.pad_w0;
        cs.dh = L.dilation_h, cs.dw = L.dilation_w, cs.group = L.group;
        cs.cg = C / L.group, cs.cgp = (L.group == 1) ? tin.cp : cs.cg;
    }
    if (work)
    {
        auto part = [&](size_t b) { return sl.nb == sl.ntot ? b : b / sl.ntot * sl.nb; }; // the slice's share of a tensor
        const size_t in_bytes = part(tin.nchw_bytes), out_bytes = part(tout.nchw_bytes);
        const double k = (double)P.k, outputs = fc ? (double)sl.nb * OC : (double)out_bytes; // an FC has one output pixel
        work->work_ops += 2.0 * outputs * k;
        work->work_bytes += (double)in_bytes + out_bytes + (double)OC * k + (L.bias ? 4.0 * OC : 0);
        work->work_wbytes += (double)OC * k + (L.bias ? 4.0 * OC : 0);
    }
    if (P.reads_nchw) s.in = g->in_nchw_dev[tin.input_index] + sl.off(tin.nchw_bytes);
    s.nhwc16 = P.nhwc16;
    if (s.kind == K_GATHER_TC)
    {
        window_plan_create(&s.wp, s.in, s.cs, s.nhwc16); // falls back to the global-memory gather (16 channels / NCHW only)
        if (!s.wp.valid && s.nhwc16 && tin.cp != 16) return fail(TB200_ERR_UNSUPPORTED, "layer %d: window plan failed for a 32-channel 3x3 convolution", li);
    }
    if (s.kind == K_CONV_DW && !(g->flags & TB200_PRERUN_NO_TENSORCORE)) dw_plan_create(&s.dwp, s.in, s.cs, s.epi); // falls back when not applicable
    if (s.kind == K_IGEMM)
    {
        int rc = gemm_plan_create_conv(&s.gemm, s.in, s.w, s.out, s.cs, P.gemm_zp);
        if (rc) return fail(rc, "layer %d: implicit-GEMM plan failed", li);
        s.gemm.fixq = g->ctx->fixq, s.gemm.fixq_cap = FIXQ_CAP;
    }
    if (s.kind == K_GEMM)
    {
        const long long m = fc ? N : (long long)N * H * W;
        const int kdim = fc ? H * W * tin.cp : tin.cp;
        int rc = gemm_plan_create(&s.gemm, s.in, kdim, s.w, s.out, m, kdim, OC, tout.cp, tout.cp, P.gemm_zp);
        if (rc) return fail(rc, "layer %d: TMA descriptor creation failed (m=%lld k=%d oc=%d)", li, m, kdim, OC);
        s.gemm.fixq = g->ctx->fixq, s.gemm.fixq_cap = FIXQ_CAP;
    }
    return 0;
}

static int fill_pool_step(const tb200_graph* g, int li, const LayerPlan& P, const Slice& sl, Step& s)
{
    const tb200_layer_desc& L = g->layers[li];
    const TensorInfo& tin = g->tensors[L.inputs[0]];
    const TensorInfo& tout = g->tensors[L.output];
    const int H = tin.d.dims[2], W = tin.d.dims[3], C = tin.d.dims[1];
    PoolShape& p = s.ps;
    p.n = sl.nb, p.h = H, p.w = W, p.c = C, p.cp = tin.cp, p.oh = tout.d.dims[2], p.ow = tout.d.dims[3];
    p.kh = L.kernel_h, p.kw = L.kernel_w, p.sh = L.stride_h, p.sw = L.stride_w, p.ph0 = L.pad_h0, p.pw0 = L.pad_w0;
    p.method = L.pool_method, p.caffe_flavor = L.caffe_flavor;
    p.in_scale = tin.d.scale, p.out_scale = tout.d.scale, p.in_zero = tin.d.zero_point, p.out_zero = tout.d.zero_point;
    if (L.pool_global) p.kh = H, p.kw = W, p.sh = p.sw = 1, p.ph0 = p.pw0 = 0;
    p.lut = P.pool_relu >= 0 ? g->w_arena + P.blob.w_off : nullptr, p.c_real = s.u8 ? C : tin.cp;
    if (tout.d.dims[1] != C) return fail(TB200_ERR_INVALID, "layer %d: pool channel mismatch", li);
    return 0;
}

// ReLU and eltwise
static int fill_pointwise_step(const tb200_graph* g, int li, const LayerPlan& P, const Slice& sl, Step& s)
{
    const tb200_layer_desc& L = g->layers[li];
    const TensorInfo& tin = g->tensors[L.inputs[0]];
    const TensorInfo& tout = g->tensors[L.output];
    PointwiseParams& p = s.pp;
    p.c = tin.d.dims[1], p.cp = tin.cp;
    p.scale0 = tin.d.scale, p.zero0 = tin.d.zero_point, p.out_scale = tout.d.scale, p.out_zero = tout.d.zero_point;
    p.negative_slope = L.negative_slope;
    p.post_relu = P.post_relu, p.post_floor4 = (uint32_t)(tout.d.zero_point & 0xff) * 0x01010101u;
    if (L.op == TB200_OP_RELU)
        p.mode = 0, p.scale1 = 0, p.zero1 = 0;
    else
    {
        const TensorInfo& t1 = g->tensors[L.inputs[1]];
        if (t1.nhwc_bytes != tin.nhwc_bytes) return fail(TB200_ERR_UNSUPPORTED, "layer %d: eltwise broadcast", li);
        p.mode = L.elt_type == TB200_ELT_SUM ? 1 : 2;
        p.scale1 = t1.d.scale, p.zero1 = t1.d.zero_point;
        s.in2 = sl.dev(t1);
    }
    s.bytes = sl.bytes(tin);
    if (tout.nhwc_bytes != tin.nhwc_bytes) return fail(TB200_ERR_INVALID, "layer %d: pointwise shape mismatch", li);
    return 0;
}

// One step per input; all but the last are pushed here, the last is left in `s`.
static int fill_concat_steps(const tb200_graph* g, int li, const LayerPlan& P, const Slice& sl, Step& s, std::vector<Step>& steps)
{
    const tb200_layer_desc& L = g->layers[li];
    const TensorInfo& tin = g->tensors[L.inputs[0]];
    const TensorInfo& tout = g->tensors[L.output];
    int coff = 0;
    for (int k = 0; k < L.num_inputs; k++)
    {
        const TensorInfo& tk = g->tensors[L.inputs[k]];
        Step p = s;
        p.in = sl.dev(tk);
        p.npix = (long long)sl.nb * tin.d.dims[2] * tin.d.dims[3], p.c = tk.d.dims[1], p.cp_in = tk.cp, p.cp_out = tout.cp, p.c_off = coff;
        p.s_in = tk.d.scale, p.z_in = tk.d.zero_point, p.s_out = tout.d.scale, p.z_out = tout.d.zero_point;
        p.c_write = (k + 1 == L.num_inputs) ? tout.cp - coff : tk.d.dims[1];
        // vectorised table path when everything is 16-channel aligned; identical quantisation -> no table at all
        p.scale = (tk.d.dims[1] % 16 == 0 && coff % 16 == 0) ? 1 : 0;
        p.w = (tk.d.scale == tout.d.scale && tk.d.zero_point == tout.d.zero_point) ? nullptr : g->w_arena + P.blob.w_off + 256 * k;
        coff += tk.d.dims[1];
        if (k + 1 < L.num_inputs) steps.push_back(p);
        else s = p;
    }
    if (coff != tout.d.dims[1]) return fail(TB200_ERR_INVALID, "layer %d: concat channels %d != %d", li, coff, tout.d.dims[1]);
    return 0;
}

// Upsample, byte table, softmax, reshape, copy.
static int fill_data_step(const tb200_graph* g, int li, const LayerPlan& P, const Slice& sl, Step& s)
{
    const tb200_layer_desc& L = g->layers[li];
    const TensorInfo& tin = g->tensors[L.inputs[0]];
    const TensorInfo& tout = g->tensors[L.output];
    const int N = sl.nb, C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3];
    const int OC = tout.d.dims[1], OH = tout.d.dims[2], OW = tout.d.dims[3];
    switch (P.kind)
    {
    case K_UPSAMPLE:
        s.n = N, s.h = H, s.w_ = W, s.cp_in = tin.cp, s.scale = L.up_scale;
        if (OH != H * L.up_scale || OW != W * L.up_scale) return fail(TB200_ERR_INVALID, "layer %d: upsample shape", li);
        break;
    case K_LUT:
        s.w = g->w_arena + P.blob.w_off;
        s.bytes = sl.bytes(tin);
        s.c = C, s.cp_in = tin.cp;
        if (tout.nhwc_bytes != tin.nhwc_bytes) return fail(TB200_ERR_INVALID, "layer %d: unary op changes the shape", li);
        break;
    case K_SOFTMAX:
        if (tout.nhwc_bytes != tin.nhwc_bytes) return fail(TB200_ERR_INVALID, "layer %d: softmax changes the shape", li);
        s.npix = (long long)N * H * W, s.c = C, s.cp_in = tin.cp;
        s.s_in = tin.d.scale, s.z_in = tin.d.zero_point, s.s_out = tout.d.scale, s.z_out = tout.d.zero_point;
        break;
    case K_RESHAPE:
        s.n = N, s.c = C, s.h = H, s.w_ = W, s.oc_ = OC, s.oh_ = OH, s.ow_ = OW;
        s.scratch = g->act_arena + P.scratch_off; // NCHW-ordered bytes of this chunk (chunks never run concurrently)
        break;
    case K_COPY:
        s.bytes = sl.bytes(tin);
        if (tout.nhwc_bytes != tin.nhwc_bytes) return fail(TB200_ERR_UNSUPPORTED, "layer %d: identity changes the NHWC footprint", li);
        break;
    }
    return 0;
}

// The launch sequence of images [first, first + nb) (the active batch, or one pipeline chunk of it) into `steps`; the work of its
// convolutions is added to *work when given.
static int build_steps(tb200_graph* g, int first, int nb, std::vector<Step>& steps, BatchPlan* work)
{
    const std::vector<LayerPlan>& plan = g->plan;
    const Slice sl{first, nb, g->tensors[0].d.dims[0]};
    auto layout_step = [&](int kind, const void* in, void* out, const TensorInfo& t)
    {
        Step s;
        s.kind = kind, s.layer = -1, s.in = in, s.out = out;
        s.n = nb, s.c = t.d.dims[1], s.h = t.d.dims[2], s.w_ = t.d.dims[3];
        steps.push_back(s);
    };
    for (size_t i = 0; i < g->input_ids.size(); i++)
    {
        const TensorInfo& t = g->tensors[g->input_ids[i]];
        if (t.nhwc_needed) layout_step(K_NCHW2NHWC, g->in_nchw_dev[i] + sl.off(t.nchw_bytes), sl.dev(t), t);
    }
    for (int li = 0; li < (int)g->layers.size(); li++)
    {
        const tb200_layer_desc& L = g->layers[li];
        const LayerPlan& P = plan[li];
        if (P.kind == K_NONE) continue; // keeps the name prerun_one gave it
        const TensorInfo& tin = g->tensors[L.inputs[0]];
        Step s;
        s.kind = P.kind, s.layer = li, s.u8 = tin.d.data_type == TB200_DT_UINT8;
        s.in = sl.dev(tin), s.out = sl.dev(g->tensors[L.output]);
        int rc;
        if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC) rc = fill_conv_step(g, li, P, sl, work, s);
        else if (P.kind == K_POOL) rc = fill_pool_step(g, li, P, sl, s);
        else if (P.kind == K_POINTWISE) rc = fill_pointwise_step(g, li, P, sl, s);
        else if (P.kind == K_CONCAT_PART) rc = fill_concat_steps(g, li, P, sl, s, steps);
        else rc = fill_data_step(g, li, P, sl, s);
        if (rc) return rc;
        g->layer_kernel[li] = (s.kind == K_CONV_DW && s.dwp.valid) ? "conv_dw3x3_tma_dp4a" : ((s.kind == K_GATHER_TC && s.wp.valid) ? "conv_window_tcgen05" : kStepName[s.kind]);
        steps.push_back(s);
    }
    for (size_t i = 0; i < g->output_ids.size(); i++)
    {
        const TensorInfo& t = g->tensors[g->output_ids[i]];
        layout_step(K_NHWC2NCHW, sl.dev(t), g->out_nchw_dev[i] + sl.off(t.nchw_bytes), t);
    }
    return 0;
}

// ---- capture the launch sequences of `bp` into CUDA graphs: [0] = whole slice, [1..K] = the pipeline chunks ----
static int capture_graphs(tb200_graph* g, BatchPlan& bp)
{
    cudaStream_t st = g->ctx->stream;
    const int ngraphs = 1 + (int)bp.chunk_steps.size();
    bp.cu_graphs.assign(ngraphs, nullptr);
    bp.cu_execs.assign(ngraphs, nullptr);
    for (int gi = 0; gi < ngraphs; gi++)
    {
        const std::vector<Step>& seq = gi == 0 ? bp.steps : bp.chunk_steps[gi - 1];
        CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        int rc = 0;
        for (const Step& s : seq)
            if ((rc = run_step(g, s, st)) != 0) break;
        cudaError_t ce = cudaStreamEndCapture(st, &bp.cu_graphs[gi]);
        if (rc) return rc;
        if (ce != cudaSuccess) return fail(TB200_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
        ce = cudaGraphInstantiate(&bp.cu_execs[gi], bp.cu_graphs[gi], 0);
        if (ce != cudaSuccess) return fail(TB200_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(ce));
    }
    // the pipeline's streams and events: made by the first plan with chunks, shared by every later one
    const int K = bp.chunks;
    if (K > 1 && !g->copy_stream)
    {
        CUDA_OK(cudaStreamCreateWithFlags(&g->copy_stream, cudaStreamNonBlocking));
        CUDA_OK(cudaStreamCreateWithFlags(&g->d2h_stream, cudaStreamNonBlocking));
        g->ev_in.resize(K), g->ev_out.resize(K);
        for (int ck = 0; ck < K; ck++)
        {
            CUDA_OK(cudaEventCreateWithFlags(&g->ev_in[ck], cudaEventDisableTiming));
            CUDA_OK(cudaEventCreateWithFlags(&g->ev_out[ck], cudaEventDisableTiming));
        }
        CUDA_OK(cudaEventCreateWithFlags(&g->ev_done, cudaEventDisableTiming));
    }
    return 0;
}

// A capture a failed CUDA call may have left open on `st` is ended and its graph dropped.
static void end_open_capture(cudaStream_t st)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone)
    {
        cudaGraph_t junk = nullptr;
        cudaStreamEndCapture(st, &junk);
        if (junk) cudaGraphDestroy(junk);
    }
    cudaGetLastError();
}

// The launch sequences of images [0, nb) of this shard into bp: the whole slice, the pipeline chunks at nb (plan_chunks) and,
// unless TB200_PRERUN_NO_GRAPH, their CUDA graphs.  nb == 0 leaves bp without steps: nothing is encoded or captured.
static int build_batch_plan(tb200_graph* g, int nb, BatchPlan& bp)
{
    bp.n = nb;
    if (nb == 0) return 0;
    // the whole-slice plan serves tb200_graph_launch / profile (device-resident use); the chunk plans serve the pipelined
    // tb200_graph_run.  They address the same tensors (a chunk is a slice of dim 0), so either may run at any time.
    plan_chunks(g, nb, bp);
    int rc;
    if ((rc = build_steps(g, 0, nb, bp.steps, &bp)) != 0) return rc;
    for (int ck = 0; ck < (int)bp.chunk_steps.size(); ck++)
        if ((rc = build_steps(g, bp.chunk_first[ck], bp.chunk_count[ck], bp.chunk_steps[ck], nullptr)) != 0) return rc;
    bp.num_launches = (int)bp.steps.size();
    for (const Step& st : bp.steps) bp.num_launches += st.kind == K_RESHAPE ? 1 : 0; // two layout kernels
    if (!(g->flags & TB200_PRERUN_NO_GRAPH) && (rc = capture_graphs(g, bp)) != 0) return rc;
    return 0;
}

// Plans one graph on one GPU.  On failure the caller destroys g (arenas, tensor maps, CUDA graphs, an open capture).
static int prerun_one(tb200_context* ctx, const tb200_tensor_desc* tensors, int num_tensors, const tb200_layer_desc* layers, int num_layers,
                      const int32_t* input_ids, int num_inputs, const int32_t* output_ids, int num_outputs, int flags, tb200_graph* g)
{
    CUDA_OK(cudaSetDevice(ctx->device));
    g->layers.assign(layers, layers + num_layers);
    g->layer_kernel.assign(num_layers, kStepName[K_NONE]); // build_steps names every layer that was not folded away
    g->plan.assign(num_layers, LayerPlan());
    std::vector<LayerPlan>& plan = g->plan;
    if (!(flags & TB200_PRERUN_NO_GRAPH)) fuse_nodes(layers, tensors, num_tensors, output_ids, num_outputs, g->layers, plan);
    int rc;
    if ((rc = setup_tensors(g, tensors, num_tensors, input_ids, num_inputs, output_ids, num_outputs)) != 0) return rc;
    if ((rc = plan_kernels(g, plan)) != 0) return rc;
    plan_activation_arena(g, plan);
    if ((rc = alloc_device_buffers(g)) != 0) return rc;
    prove_fast_epilogues(g, plan);
    if (!(flags & TB200_PRERUN_NO_WEIGHTS) && (rc = upload_weights(g, plan)) != 0) return rc;
    CUDA_OK(cudaStreamSynchronize(ctx->stream));
    g->cur = &g->prepared;
    return build_batch_plan(g, g->tensors[0].d.dims[0], g->prepared);
}

// ---- page-locking of the caller's buffers ---------------------------------------------------------------------------------
// Tengine hands `run` the application's malloc'd NCHW buffers (ir_tensor->data, c_api.c:1141-1160).  A cudaMemcpyAsync from
// pageable memory is staged by the driver and blocks the calling thread, which would serialise the GPUs of a group and the
// chunks of the copy/compute pipeline.  So a buffer is registered (cudaHostRegisterPortable) the first time it is seen and the
// registration is cached (up to 16 ranges, oldest dropped; everything is unregistered at postrun / context destruction).
// Returns true when [p, p+bytes) is page-locked.  Failure is not an error: the copy then takes the driver's pageable path.
static bool host_pin(tb200_context* root, const void* ptr, size_t bytes)
{
    if (!ptr || !bytes) return false;
    const uint8_t* p = (const uint8_t*)ptr;
    for (const HostReg& r : root->host_regs)
        if (p >= r.p && p + bytes <= r.p + r.bytes) return true;
    for (const void* f : root->host_reg_failed)
        if (f == ptr) return false;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, ptr) == cudaSuccess && at.type == cudaMemoryTypeHost)
    {
        root->host_regs.push_back(HostReg{p, bytes, false}); // already page-locked by its owner
        return true;
    }
    cudaGetLastError();
    // an older, smaller registration of the same buffer would make the new one fail: drop overlapping ranges of ours first
    for (size_t i = 0; i < root->host_regs.size();)
    {
        const HostReg& r = root->host_regs[i];
        if (r.ours && p < r.p + r.bytes && r.p < p + bytes)
        {
            if (cudaHostUnregister((void*)r.p) != cudaSuccess) cudaGetLastError();
            root->host_regs.erase(root->host_regs.begin() + i);
        }
        else
            i++;
    }
    if (cudaHostRegister((void*)ptr, bytes, cudaHostRegisterPortable) != cudaSuccess)
    {
        cudaGetLastError();
        if (root->host_reg_failed.size() < 64) root->host_reg_failed.push_back(ptr);
        return false;
    }
    root->host_regs.push_back(HostReg{p, bytes, true});
    if (root->host_regs.size() > 16)
    {
        if (root->host_regs[0].ours && cudaHostUnregister((void*)root->host_regs[0].p) != cudaSuccess) cudaGetLastError();
        root->host_regs.erase(root->host_regs.begin());
    }
    return true;
}


// every shard of a graph, the root's own first
template <typename F>
static int for_each_shard(tb200_graph* g, F f)
{
    int rc = f(g, 0);
    for (size_t i = 0; rc == 0 && i < g->shards.size(); i++) rc = f(g->shards[i], (int)i + 1);
    return rc;
}
// the shards that hold images of the active batch: a shard left without any issues no copy, kernel or graph launch
template <typename F>
static int for_each_busy_shard(tb200_graph* g, F f)
{
    return for_each_shard(g, [&](tb200_graph* sh, int r) { return sh->num_images ? f(sh, r) : 0; });
}
// NCHW bytes of one image of a tensor (from the batch of prerun, which sized the tensor)
static inline size_t image_bytes(const tb200_graph* g, int tensor_id) { return g->tensors[tensor_id].nchw_bytes / (size_t)g->prep_images; }
// dim 0 and NCHW bytes of the shard's active images of a tensor: all of it at the batch of prerun (also when its dim 0 is not the
// batch), else num_images images
static inline int active_dim0(const tb200_graph* g, const TensorInfo& t) { return g->num_images == g->prep_images ? t.d.dims[0] : g->num_images; }
static inline size_t active_nchw_bytes(const tb200_graph* g, const TensorInfo& t)
{
    return g->num_images == g->prep_images ? t.nchw_bytes : t.nchw_bytes / (size_t)t.d.dims[0] * (size_t)g->num_images;
}

// One ncclBroadcast of the packed arena from GPU 0 to every other GPU of the group (grouped: one call per device from this
// single thread), or peer copies when NCCL is not in use.
static int broadcast_arena(tb200_graph* g)
{
    tb200_context* root = g->ctx;
    if (g->shards.empty()) return 0;
    CUDA_OK(cudaSetDevice(root->device));
    CUDA_OK(cudaStreamSynchronize(root->stream));
    NcclApi* nc = root->comms.empty() ? nullptr : nccl_api();
    if (nc)
    {
        STAGE("grouped ncclBroadcast of %zu bytes ...", g->w_bytes);
        int r = nc->GroupStart();
        if (r == 0) r = nc->Broadcast(g->w_arena, g->w_arena, g->w_bytes, /*ncclUint8*/ 1, 0, root->comms[0], root->stream);
        for (size_t i = 0; r == 0 && i < g->shards.size(); i++)
        {
            tb200_graph* sh = g->shards[i];
            if (sh->w_bytes != g->w_bytes) return fail(TB200_ERR_INVALID, "shard %d planned a different weight arena (%zu vs %zu bytes)", (int)i + 1, sh->w_bytes, g->w_bytes);
            r = nc->Broadcast(sh->w_arena, sh->w_arena, sh->w_bytes, 1, 0, root->comms[i + 1], sh->ctx->stream);
        }
        const int r2 = nc->GroupEnd();
        STAGE("ncclGroupEnd -> %d / %d", r, r2);
        if (r || r2) return fail(TB200_ERR_CUDA, "ncclBroadcast of the weight arena failed: %s", nc->GetErrorString(r ? r : r2));
    }
    else
    {
        for (size_t i = 0; i < g->shards.size(); i++)
        {
            tb200_graph* sh = g->shards[i];
            if (sh->w_bytes != g->w_bytes) return fail(TB200_ERR_INVALID, "shard %d planned a different weight arena", (int)i + 1);
            CUDA_OK(cudaMemcpyPeerAsync(sh->w_arena, sh->ctx->device, g->w_arena, root->device, g->w_bytes, root->stream));
        }
    }
    CUDA_OK(cudaSetDevice(root->device));
    CUDA_OK(cudaStreamSynchronize(root->stream));
    STAGE("broadcast: root stream drained");
    for (tb200_graph* sh : g->shards)
    {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        CUDA_OK(cudaStreamSynchronize(sh->ctx->stream));
    }
    CUDA_OK(cudaSetDevice(root->device));
    return 0;
}

static int prerun_guarded(tb200_context* ctx, const tb200_tensor_desc* tensors, int num_tensors, const tb200_layer_desc* layers, int num_layers,
                          const int32_t* input_ids, int num_inputs, const int32_t* output_ids, int num_outputs, int flags, tb200_graph** out)
{
    tb200_graph* g = new tb200_graph();
    g->ctx = ctx, g->flags = flags;
    const int rc = prerun_one(ctx, tensors, num_tensors, layers, num_layers, input_ids, num_inputs, output_ids, num_outputs, flags, g);
    if (rc)
    {
        end_open_capture(ctx->stream);
        destroy_graph(g);
        return rc;
    }
    g->num_images = g->prep_images = g->total_images = g->batch = tensors[0].dims[0];
    *out = g;
    return 0;
}

extern "C" {

int tb200_graph_prerun(tb200_context* ctx, const tb200_tensor_desc* tensors, int num_tensors, const tb200_layer_desc* layers, int num_layers,
                       const int32_t* input_ids, int num_inputs, const int32_t* output_ids, int num_outputs, int flags, tb200_graph** out)
{
    if (!ctx || !tensors || !layers || !out || num_tensors <= 0 || num_layers <= 0) return fail(TB200_ERR_INVALID, "bad arguments");
    if ((num_inputs > 0 && !input_ids) || (num_outputs > 0 && !output_ids)) return fail(TB200_ERR_INVALID, "null id table");
    // ---- how many GPUs take part: the batch (dim 0, the same for every tensor) is cut into contiguous slices ----
    int R = 1 + (int)ctx->peers.size();
    const int N = tensors[0].dims[0];
    for (int i = 0; i < num_tensors; i++)
        if (tensors[i].dims[0] != N) R = 1; // not a plain batch dimension: GPU 0 runs the whole subgraph
    if (R > N) R = N > 0 ? N : 1;
    if (R == 1) return prerun_guarded(ctx, tensors, num_tensors, layers, num_layers, input_ids, num_inputs, output_ids, num_outputs, flags, out);

    std::vector<tb200_tensor_desc> td(tensors, tensors + num_tensors);
    tb200_graph* root = nullptr;
    int first = 0;
    for (int r = 0; r < R; r++)
    {
        int count = 0;
        tb200_shard_range(N, R, r, nullptr, &count);
        for (auto& t : td) t.dims[0] = count;
        tb200_graph* sh = nullptr;
        tb200_context* c = r == 0 ? ctx : ctx->peers[r - 1];
        // GPU 0 packs the weights; the others only allocate the arena (same layout: it depends on the descriptors alone)
        const int rc = prerun_guarded(c, td.data(), num_tensors, layers, num_layers, input_ids, num_inputs, output_ids, num_outputs,
                                      flags | (r ? TB200_PRERUN_NO_WEIGHTS : 0), &sh);
        if (rc)
        {
            if (root) destroy_graph(root);
            cudaSetDevice(ctx->device);
            return rc;
        }
        sh->first_image = first, sh->num_images = sh->prep_images = count, sh->total_images = sh->batch = N;
        first += count;
        if (r == 0) root = sh;
        else root->shards.push_back(sh);
    }
    if (!(flags & TB200_PRERUN_NO_WEIGHTS))
    {
        const int rc = broadcast_arena(root);
        if (rc)
        {
            destroy_graph(root);
            return rc;
        }
    }
    cudaSetDevice(ctx->device);
    *out = root;
    return 0;
}

// how a batch of n images is cut over `world` GPUs: contiguous slices of dim 0, the first n % world shards one image longer
int tb200_shard_range(int n_images, int world, int rank, int* first_image, int* num_images)
{
    if (n_images < 0 || world < 1 || rank < 0 || rank >= world) return fail(TB200_ERR_INVALID, "bad shard arguments");
    const int base = n_images / world, extra = n_images % world;
    if (first_image) *first_image = rank * base + (rank < extra ? rank : extra);
    if (num_images) *num_images = base + (rank < extra ? 1 : 0);
    return 0;
}

int tb200_graph_broadcast_weights(tb200_graph* g)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    return broadcast_arena(g);
}

int tb200_probe_int8_tops(tb200_context* ctx, double* tops)
{
    if (!ctx || !tops) return fail(TB200_ERR_INVALID, "bad arguments");
    CUDA_OK(cudaSetDevice(ctx->device));
    const cudaError_t e = probe_int8_mma_peak(ctx->num_sms, tops, ctx->stream);
    if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "int8 MMA probe: %s", cudaGetErrorString(e));
    return 0;
}

int tb200_pack_cache_dir(const char* dir)
{
    g_pack_cache_set = true;
    g_pack_cache_dir = dir ? dir : "";
    return 0;
}
int tb200_graph_pack_cache_state(tb200_graph* g) { return g ? g->pack_cache_state : 0; }

int tb200_graph_num_shards(tb200_graph* g) { return g ? 1 + (int)g->shards.size() : 0; }

int tb200_graph_shard(tb200_graph* g, int index, int* cuda_device, int* first_image, int* num_images)
{
    if (!g || index < 0 || index > (int)g->shards.size()) return fail(TB200_ERR_INVALID, "shard index out of range");
    const tb200_graph* sh = index == 0 ? g : g->shards[index - 1];
    if (cuda_device) *cuda_device = sh->ctx->device;
    if (first_image) *first_image = sh->first_image;
    if (num_images) *num_images = sh->num_images;
    return 0;
}

// Drains every stream of every shard, then makes images [0, n) the batch of every later call.  The steps and CUDA graphs of a
// batch other than the prepared one are built once and kept until another such batch replaces them.
int tb200_graph_set_batch(tb200_graph* g, int n)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    if (n < 1 || n > g->total_images) return fail(TB200_ERR_INVALID, "set_batch: %d images; the graph was prepared for 1..%d", n, g->total_images);
    if (n == g->batch) return 0;
    for (const TensorInfo& t : g->tensors)
        if (t.d.dims[0] != g->tensors[0].d.dims[0])
            return fail(TB200_ERR_UNSUPPORTED, "set_batch: the graph's tensors differ in dim 0, so it runs only at the batch of %d it was prepared for",
                        g->total_images);
    int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        if (sh->copy_stream) CUDA_OK(cudaStreamSynchronize(sh->copy_stream));
        if (sh->d2h_stream) CUDA_OK(cudaStreamSynchronize(sh->d2h_stream));
        CUDA_OK(cudaStreamSynchronize(sh->ctx->stream));
        return 0;
    });
    const int R = 1 + (int)g->shards.size();
    auto shard = [&](int r) { return r == 0 ? g : g->shards[r - 1]; };
    const bool prepared = n == g->total_images;
    if (rc == 0 && !prepared && n != g->other_batch)
    {
        // build every shard's plan before replacing any: a failure leaves the graph as it was
        std::vector<BatchPlan> fresh(R);
        for (int r = 0; r < R && rc == 0; r++)
        {
            tb200_graph* sh = shard(r);
            int count = 0;
            tb200_shard_range(n, R, r, nullptr, &count);
            const std::vector<const char*> names = sh->layer_kernel; // the kernel names stay those of prerun
            cudaSetDevice(sh->ctx->device);
            rc = build_batch_plan(sh, count, fresh[r]);
            sh->layer_kernel = names;
            if (rc) end_open_capture(sh->ctx->stream);
        }
        for (int r = 0; r < R; r++)
        {
            tb200_graph* sh = shard(r);
            cudaSetDevice(sh->ctx->device);
            destroy_batch_plan(rc ? fresh[r] : sh->other);
            if (!rc) sh->other = std::move(fresh[r]);
        }
        if (!rc) g->other_batch = n;
    }
    if (rc == 0)
        for (int r = 0; r < R; r++)
        {
            tb200_graph* sh = shard(r);
            sh->cur = prepared ? &sh->prepared : &sh->other;
            tb200_shard_range(n, R, r, &sh->first_image, &sh->num_images);
            sh->batch = n;
        }
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_batch(tb200_graph* g)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    return g->batch;
}

int tb200_graph_arena_bytes(tb200_graph* g, size_t* activation_bytes, size_t* unshared_bytes, size_t* weight_bytes)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    if (activation_bytes) *activation_bytes = g->act_bytes;
    if (unshared_bytes) *unshared_bytes = g->act_unshared_bytes;
    if (weight_bytes) *weight_bytes = g->w_bytes;
    return 0;
}

int tb200_graph_upload(tb200_graph* g, int input_index, const void* host_nchw)
{
    if (!g || input_index < 0 || input_index >= (int)g->input_ids.size() || !host_nchw) return fail(TB200_ERR_INVALID, "bad upload arguments");
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const int id = sh->input_ids[input_index];
        CUDA_OK(host_copy(g->ctx, sh->in_nchw_dev[input_index], (const uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, id),
                                active_nchw_bytes(sh, sh->tensors[id]), cudaMemcpyHostToDevice, sh->ctx->stream));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

// Checks shared by the image upload entry points: every descriptor of the batch names a 3- or 4-channel image of 2..32767 pixels a side
// inside the buffer, and mean / scale are finite.  `what` names the entry point in the message.
static int check_images(const tb200_graph* g, const char* what, size_t pixel_bytes, const tb200_image* images, const float* mean, const float* scale)
{
    for (int k = 0; k < 3; k++)
        if (!std::isfinite(mean[k]) || !std::isfinite(scale[k])) return fail(TB200_ERR_INVALID, "%s: mean / scale %d is not finite", what, k);
    for (int i = 0; i < g->batch; i++)
    {
        const tb200_image& im = images[i];
        if (im.c != 3 && im.c != 4) return fail(TB200_ERR_UNSUPPORTED, "%s: image %d has %d channels (3 or 4 supported)", what, i, im.c);
        if (im.w < 2 || im.h < 2 || im.w > 32767 || im.h > 32767) return fail(TB200_ERR_INVALID, "%s: image %d is %d x %d (2..32767)", what, i, im.w, im.h);
        const uint64_t bytes = (uint64_t)im.w * (uint64_t)im.h * (uint64_t)im.c;
        if (im.offset > pixel_bytes || bytes > pixel_bytes - im.offset)
            return fail(TB200_ERR_INVALID, "%s: image %d (offset %llu, %llu bytes) lies outside the %zu-byte pixel buffer", what, i, (unsigned long long)im.offset,
                        (unsigned long long)bytes, pixel_bytes);
    }
    return 0;
}

// Every shard copies the byte span of its own images (in whatever order they lie in the caller's buffer) and their descriptors, then
// `launch(shard, staged pixels, descriptors, n, stream)` fills the shard's NCHW input buffer -- the buffer tb200_graph_upload fills -- so
// the captured graph runs as is.  geo: per image of the batch the detection geometry the descriptors carry, or null.
extern "C++" {
template <typename Launch>
static int upload_staged_images(tb200_graph* g, const char* what, const void* pixels, size_t pixel_bytes, const tb200_image* images,
                                const tb200_detect_geometry* geo, Launch launch)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    host_pin(g->ctx, pixels, pixel_bytes);
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        cudaGetLastError(); // the launch below reports cudaGetLastError(): a non-sticky error an earlier call left behind is not its own
        const int n = sh->num_images;
        const tb200_image* im = images + sh->first_image;
        const tb200_detect_geometry* gm = geo ? geo + sh->first_image : nullptr;
        uint64_t lo = UINT64_MAX, hi = 0;
        for (int i = 0; i < n; i++)
            lo = std::min(lo, im[i].offset), hi = std::max(hi, im[i].offset + (uint64_t)im[i].w * im[i].h * im[i].c);
        if (hi - lo > sh->img_stage_bytes)
        {
            cudaFree(sh->img_stage);
            sh->img_stage = nullptr, sh->img_stage_bytes = 0;
            CUDA_OK(cudaMalloc(&sh->img_stage, hi - lo));
            sh->img_stage_bytes = hi - lo;
        }
        if (!sh->img_ev) CUDA_OK(cudaEventCreateWithFlags(&sh->img_ev, cudaEventDisableTiming));
        CUDA_OK(cudaEventSynchronize(sh->img_ev)); // the previous descriptor copy has read the host staging
        if (n > sh->img_desc_cap)
        {
            cudaFree(sh->img_desc), cudaFreeHost(sh->img_desc_host);
            sh->img_desc = sh->img_desc_host = nullptr, sh->img_desc_cap = 0;
            CUDA_OK(cudaMalloc(&sh->img_desc, sizeof(ImageDesc) * n));
            CUDA_OK(cudaHostAlloc(&sh->img_desc_host, sizeof(ImageDesc) * n, cudaHostAllocDefault));
            sh->img_desc_cap = n;
        }
        for (int i = 0; i < n; i++)
            sh->img_desc_host[i] = gm ? ImageDesc{im[i].offset - lo, im[i].w, im[i].h, im[i].c, gm[i].resize_w, gm[i].resize_h, gm[i].left, gm[i].top}
                                      : ImageDesc{im[i].offset - lo, im[i].w, im[i].h, im[i].c, 0, 0, 0, 0};
        cudaStream_t st = sh->ctx->stream;
        CUDA_OK(host_copy(g->ctx, sh->img_stage, (const uint8_t*)pixels + lo, hi - lo, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaMemcpyAsync(sh->img_desc, sh->img_desc_host, sizeof(ImageDesc) * n, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaEventRecord(sh->img_ev, st));
        const cudaError_t e = launch(sh, sh->img_stage, sh->img_desc, n, st);
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "%s: launch of its kernel failed: %s", what, cudaGetErrorString(e));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}
} // extern "C++"

int tb200_graph_upload_images(tb200_graph* g, int input_index, const void* pixels, size_t pixel_bytes, const tb200_image* images, const float mean[3],
                              const float scale[3])
{
    static_assert(offsetof(ImageDesc, w) == offsetof(tb200_image, w) && offsetof(ImageDesc, c) == offsetof(tb200_image, c), "image descriptor layout");
    if (!g || !pixels || !images || !mean || !scale || input_index < 0 || input_index >= (int)g->input_ids.size())
        return fail(TB200_ERR_INVALID, "bad upload_images arguments");
    const tb200_tensor_desc& td = g->tensors[g->input_ids[input_index]].d;
    if (td.dims[1] != 3) return fail(TB200_ERR_INVALID, "upload_images: input %d has %d channels, not 3", input_index, td.dims[1]);
    if (td.data_type != TB200_DT_INT8 && td.data_type != TB200_DT_UINT8) return fail(TB200_ERR_INVALID, "upload_images: input %d is not int8 / uint8", input_index);
    if (const int rc = check_images(g, "upload_images", pixel_bytes, images, mean, scale)) return rc;
    const bool u8 = td.data_type == TB200_DT_UINT8;
    return upload_staged_images(g, "upload_images", pixels, pixel_bytes, images, nullptr,
                                [&](tb200_graph* sh, const uint8_t* px, const ImageDesc* desc, int n, cudaStream_t st) {
                                    return launch_image_pre(px, desc, n, sh->in_nchw_dev[input_index], td.dims[2], td.dims[3], mean, scale, td.scale,
                                                            td.zero_point, u8, st);
                                });
}

// Where an image of src_w x src_h lands in the W x H laid-out input: stretch fills it; letterbox restates examples/tm_yolov5s.cpp:274-295
// (the scale compared in double and kept in float, the resized size a float product truncated, the borders halved downwards).
static tb200_detect_geometry detect_geometry(int mode, int src_w, int src_h, int W, int H)
{
    tb200_detect_geometry r{src_w, src_h, W, H, 0, 0, 0.f};
    if (mode == TB200_PRE_STRETCH) return r;
    float scale_letterbox;
    if ((H * 1.0 / src_h) < (W * 1.0 / src_w))
        scale_letterbox = H * 1.0 / src_h;
    else
        scale_letterbox = W * 1.0 / src_w;
    r.resize_w = int(scale_letterbox * (float)src_w);
    r.resize_h = int(scale_letterbox * (float)src_h);
    r.left = (W - r.resize_w) / 2, r.top = (H - r.resize_h) / 2;
    r.scale = scale_letterbox;
    return r;
}

int tb200_graph_upload_detect_images(tb200_graph* g, int input_index, const void* pixels, size_t pixel_bytes, const tb200_image* images,
                                     const tb200_detect_pre* pre, tb200_detect_geometry* geometry_out)
{
    if (!g || !pixels || !images || !pre || input_index < 0 || input_index >= (int)g->input_ids.size())
        return fail(TB200_ERR_INVALID, "bad upload_detect_images arguments");
    if (pre->mode != TB200_PRE_STRETCH && pre->mode != TB200_PRE_LETTERBOX) return fail(TB200_ERR_INVALID, "upload_detect_images: mode %d", pre->mode);
    if (pre->focus != 0 && pre->focus != 1) return fail(TB200_ERR_INVALID, "upload_detect_images: focus %d (0 or 1)", pre->focus);
    const tb200_tensor_desc& td = g->tensors[g->input_ids[input_index]].d;
    const bool focus = pre->focus == 1;
    if (td.dims[1] != (focus ? 12 : 3))
        return fail(TB200_ERR_INVALID, "upload_detect_images: input %d has %d channels, not %d", input_index, td.dims[1], focus ? 12 : 3);
    if (td.data_type != TB200_DT_INT8 && td.data_type != TB200_DT_UINT8)
        return fail(TB200_ERR_INVALID, "upload_detect_images: input %d is not int8 / uint8", input_index);
    // the laid-out image: the input's own H x W, or twice it with Focus
    const int H = focus ? td.dims[2] * 2 : td.dims[2], W = focus ? td.dims[3] * 2 : td.dims[3];
    if (const int rc = check_images(g, "upload_detect_images", pixel_bytes, images, pre->mean, pre->scale)) return rc;
    std::vector<tb200_detect_geometry> geo(g->batch);
    for (int i = 0; i < g->batch; i++)
    {
        geo[i] = detect_geometry(pre->mode, images[i].w, images[i].h, W, H);
        if (geo[i].resize_w < 1 || geo[i].resize_h < 1 || geo[i].resize_w > W || geo[i].resize_h > H)
            return fail(TB200_ERR_INVALID, "upload_detect_images: image %d (%d x %d) letterboxes to %d x %d in %d x %d", i, images[i].w, images[i].h,
                        geo[i].resize_w, geo[i].resize_h, W, H);
    }
    const bool u8 = td.data_type == TB200_DT_UINT8;
    const int rc = upload_staged_images(g, "upload_detect_images", pixels, pixel_bytes, images, geo.data(),
                                        [&](tb200_graph* sh, const uint8_t* px, const ImageDesc* desc, int n, cudaStream_t st) {
                                            return launch_detect_pre(px, desc, n, sh->in_nchw_dev[input_index], H, W, focus, pre->mean, pre->scale, td.scale,
                                                                     td.zero_point, u8, st);
                                        });
    if (rc == 0 && geometry_out) std::copy(geo.begin(), geo.end(), geometry_out);
    return rc;
}

// examples/tm_yolov3_tiny_uint8.cpp:501-532 (stretch) / tm_yolov5s.cpp:580-625 (letterbox), one box at a time, in float as there
static void box_to_source(int mode, const tb200_detect_geometry& gm, tb200_detection& d)
{
    float x0 = d.x, y0 = d.y, x1 = d.x + d.w, y1 = d.y + d.h;
    if (mode == TB200_PRE_STRETCH)
    {
        const float ratio_x = (float)gm.src_w / gm.resize_w, ratio_y = (float)gm.src_h / gm.resize_h;
        x0 = x0 * ratio_x, y0 = y0 * ratio_y, x1 = x1 * ratio_x, y1 = y1 * ratio_y;
    }
    else
    {
        const float ratio_x = (float)gm.src_h / gm.resize_h, ratio_y = (float)gm.src_w / gm.resize_w; // rows for x: the example's own
        x0 = (x0 - gm.left) * ratio_x, y0 = (y0 - gm.top) * ratio_y;
        x1 = (x1 - gm.left) * ratio_x, y1 = (y1 - gm.top) * ratio_y;
    }
    x0 = std::max(std::min(x0, (float)(gm.src_w - 1)), 0.f);
    y0 = std::max(std::min(y0, (float)(gm.src_h - 1)), 0.f);
    x1 = std::max(std::min(x1, (float)(gm.src_w - 1)), 0.f);
    y1 = std::max(std::min(y1, (float)(gm.src_h - 1)), 0.f);
    d.x = x0, d.y = y0, d.w = x1 - x0, d.h = y1 - y0;
}

int tb200_detections_to_source(int mode, const tb200_detect_geometry* geometry, int num_images, tb200_detection* dets, int max_per_image,
                               const int32_t* counts)
{
    if (mode != TB200_PRE_STRETCH && mode != TB200_PRE_LETTERBOX) return fail(TB200_ERR_INVALID, "detections_to_source: mode %d", mode);
    if (num_images < 0 || max_per_image < 1 || (num_images > 0 && (!geometry || !dets || !counts)))
        return fail(TB200_ERR_INVALID, "bad detections_to_source arguments");
    for (int i = 0; i < num_images; i++)
    {
        const tb200_detect_geometry& gm = geometry[i];
        if (counts[i] > max_per_image) return fail(TB200_ERR_INVALID, "detections_to_source: image %d has %d boxes, more than %d", i, counts[i], max_per_image);
        if (gm.src_w < 1 || gm.src_h < 1 || gm.resize_w < 1 || gm.resize_h < 1)
            return fail(TB200_ERR_INVALID, "detections_to_source: image %d has geometry %d x %d -> %d x %d", i, gm.src_w, gm.src_h, gm.resize_w, gm.resize_h);
    }
    for (int i = 0; i < num_images; i++)
        for (int k = 0; k < counts[i]; k++) box_to_source(mode, geometry[i], dets[(size_t)i * max_per_image + k]);
    return 0;
}

static int launch_one(tb200_graph* g)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    static const int dbg = getenv("TB200_DEBUG_HASH") ? atoi(getenv("TB200_DEBUG_HASH")) : 0;
    if (dbg >= 2)
    {
        // debug: launch by launch, a hash of every layer's output tensor (NHWC bytes) and of the weight arena
        std::vector<uint8_t> host;
        host.resize(g->w_bytes);
        CUDA_OK(cudaMemcpy(host.data(), g->w_arena, g->w_bytes, cudaMemcpyDeviceToHost));
        fprintf(stderr, "[tb200 dbg] weight arena %zu bytes hash %016llx\n", g->w_bytes, (unsigned long long)fnv1a(host.data(), g->w_bytes));
        for (const Step& s : g->cur->steps)
        {
            int rc = run_step(g, s, g->ctx->stream);
            if (rc) return rc;
            CUDA_OK(cudaStreamSynchronize(g->ctx->stream));
            if (s.layer < 0) continue;
            const TensorInfo& t = g->tensors[g->layers[s.layer].output];
            host.resize(t.nhwc_bytes);
            CUDA_OK(cudaMemcpy(host.data(), t.dev, t.nhwc_bytes, cudaMemcpyDeviceToHost));
            fprintf(stderr, "[tb200 dbg] layer %d %s out [%d %d %d %d] hash %016llx\n", s.layer, kStepName[s.kind], t.d.dims[0], t.d.dims[1], t.d.dims[2], t.d.dims[3],
                    (unsigned long long)fnv1a(host.data(), t.nhwc_bytes));
        }
        return 0;
    }
    if (!g->cur->cu_execs.empty())
    {
        CUDA_OK(cudaGraphLaunch(g->cur->cu_execs[0], g->ctx->stream)); // the whole-batch graph
        return 0;
    }
    for (const Step& s : g->cur->steps)
    {
        int rc = run_step(g, s, g->ctx->stream);
        if (rc) return rc;
    }
    return 0;
}

int tb200_graph_launch(tb200_graph* g)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) { return launch_one(sh); });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_download(tb200_graph* g, int output_index, void* host_nchw)
{
    if (!g || output_index < 0 || output_index >= (int)g->output_ids.size() || !host_nchw) return fail(TB200_ERR_INVALID, "bad download arguments");
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const int id = sh->output_ids[output_index];
        CUDA_OK(host_copy(g->ctx, (uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, id), sh->out_nchw_dev[output_index],
                                active_nchw_bytes(sh, sh->tensors[id]), cudaMemcpyDeviceToHost, sh->ctx->stream));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_sync(tb200_graph* g)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        CUDA_OK(cudaStreamSynchronize(sh->ctx->stream));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

// ---- run: three phases over the shards so that every GPU's copy engine starts before any GPU's kernels are queued ----
// (1) queue the H2D copies of all chunks on the shard's copy stream
static int run_enqueue_h2d(tb200_context* root, tb200_graph* g, const void* const* host_inputs)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    if (g->cur->chunks <= 1 || g->cur->cu_execs.empty())
    {
        for (size_t i = 0; i < g->input_ids.size(); i++)
        {
            const int id = g->input_ids[i];
            CUDA_OK(host_copy(root, g->in_nchw_dev[i], (const uint8_t*)host_inputs[i] + (size_t)g->first_image * image_bytes(g, id),
                                    active_nchw_bytes(g, g->tensors[id]), cudaMemcpyHostToDevice, g->ctx->stream));
        }
        return 0;
    }
    // Pipelined: the H2D copies of all chunks are queued back to back on the copy stream (the link stays busy), chunk k's
    // kernels start as soon as ITS slice has landed, and its outputs leave on a third stream while chunk k+1 computes.
    const int K = g->cur->chunks;
    CUDA_OK(cudaEventRecord(g->ev_done, g->ctx->stream)); // order after whatever the caller queued on the context stream
    CUDA_OK(cudaStreamWaitEvent(g->copy_stream, g->ev_done, 0));
    for (int ck = 0; ck < K; ck++)
    {
        for (size_t i = 0; i < g->input_ids.size(); i++)
        {
            const int id = g->input_ids[i];
            const size_t ib = image_bytes(g, id), off = ib * (size_t)g->cur->chunk_first[ck], bytes = ib * (size_t)g->cur->chunk_count[ck];
            CUDA_OK(host_copy(root, g->in_nchw_dev[i] + off, (const uint8_t*)host_inputs[i] + (size_t)g->first_image * ib + off, bytes, cudaMemcpyHostToDevice,
                                    g->copy_stream));
        }
        CUDA_OK(cudaEventRecord(g->ev_in[ck], g->copy_stream));
    }
    return 0;
}
// (2) kernels + D2H
static int run_enqueue_compute(tb200_context* root, tb200_graph* g, void* const* host_outputs)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    cudaStream_t cs = g->ctx->stream;
    static const int dbg2 = getenv("TB200_DEBUG_HASH") ? atoi(getenv("TB200_DEBUG_HASH")) : 0;
    if (g->cur->chunks <= 1 || g->cur->cu_execs.empty() || dbg2 >= 2)
    {
        int rc = launch_one(g);
        if (rc) return rc;
        for (size_t i = 0; i < g->output_ids.size(); i++)
        {
            const int id = g->output_ids[i];
            CUDA_OK(host_copy(root, (uint8_t*)host_outputs[i] + (size_t)g->first_image * image_bytes(g, id), g->out_nchw_dev[i], active_nchw_bytes(g, g->tensors[id]),
                                    cudaMemcpyDeviceToHost, cs));
        }
        return 0;
    }
    const int K = g->cur->chunks;
    for (int ck = 0; ck < K; ck++)
    {
        CUDA_OK(cudaStreamWaitEvent(cs, g->ev_in[ck], 0));
        CUDA_OK(cudaGraphLaunch(g->cur->cu_execs[1 + ck], cs));
        CUDA_OK(cudaEventRecord(g->ev_out[ck], cs));
        CUDA_OK(cudaStreamWaitEvent(g->d2h_stream, g->ev_out[ck], 0));
        for (size_t i = 0; i < g->output_ids.size(); i++)
        {
            const int id = g->output_ids[i];
            const size_t ib = image_bytes(g, id), off = ib * (size_t)g->cur->chunk_first[ck], bytes = ib * (size_t)g->cur->chunk_count[ck];
            CUDA_OK(host_copy(root, (uint8_t*)host_outputs[i] + (size_t)g->first_image * ib + off, g->out_nchw_dev[i] + off, bytes, cudaMemcpyDeviceToHost,
                                    g->d2h_stream));
        }
    }
    return 0;
}
// (3) wait
static int run_wait(tb200_graph* g)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    if (g->d2h_stream && g->cur->chunks > 1 && !g->cur->cu_execs.empty()) CUDA_OK(cudaStreamSynchronize(g->d2h_stream));
    CUDA_OK(cudaStreamSynchronize(g->ctx->stream));
    return 0;
}

int tb200_graph_run(tb200_graph* g, const void* const* host_inputs, void* const* host_outputs)
{
    if (!g || !host_inputs || !host_outputs) return fail(TB200_ERR_INVALID, "bad run arguments");
    for (size_t i = 0; i < g->input_ids.size(); i++)
        if (!host_inputs[i]) return fail(TB200_ERR_INVALID, "run: input %d has no host buffer", (int)i);
    for (size_t i = 0; i < g->output_ids.size(); i++)
        if (!host_outputs[i]) return fail(TB200_ERR_INVALID, "run: output %d has no host buffer (the graph has %d outputs)", (int)i, (int)g->output_ids.size());
    // page-lock the caller's buffers (whole batch) on first sight
    CUDA_OK(cudaSetDevice(g->ctx->device));
    for (size_t i = 0; i < g->input_ids.size(); i++) host_pin(g->ctx, host_inputs[i], image_bytes(g, g->input_ids[i]) * (size_t)g->batch);
    for (size_t i = 0; i < g->output_ids.size(); i++) host_pin(g->ctx, host_outputs[i], image_bytes(g, g->output_ids[i]) * (size_t)g->batch);
    int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) { return run_enqueue_h2d(g->ctx, sh, host_inputs); });
    if (!rc) rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) { return run_enqueue_compute(g->ctx, sh, host_outputs); });
    const int rc2 = for_each_shard(g, [&](tb200_graph* sh, int) { return run_wait(sh); }); // always drain what was queued
    cudaSetDevice(g->ctx->device);
    static const bool dbg = getenv("TB200_DEBUG_HASH") != nullptr;
    if (dbg)
    {
        for (size_t i = 0; i < g->input_ids.size(); i++)
            fprintf(stderr, "[tb200 run] input %zu: %zu bytes, hash %016llx\n", i, image_bytes(g, g->input_ids[i]) * (size_t)g->batch,
                    (unsigned long long)fnv1a(host_inputs[i], image_bytes(g, g->input_ids[i]) * (size_t)g->batch));
        for (size_t i = 0; i < g->output_ids.size(); i++)
            fprintf(stderr, "[tb200 run] output %zu (tensor %d): %zu bytes, hash %016llx\n", i, g->output_ids[i], image_bytes(g, g->output_ids[i]) * (size_t)g->batch,
                    (unsigned long long)fnv1a(host_outputs[i], image_bytes(g, g->output_ids[i]) * (size_t)g->batch));
        fprintf(stderr, "[tb200 run] %zu layers, %d launches, chunks %d, shards %zu, flags %d\n", g->layers.size(), g->cur->num_launches, g->cur->chunks, g->shards.size() + 1, g->flags);
    }
    return rc ? rc : rc2;
}

int tb200_graph_postrun(tb200_graph* g)
{
    if (!g) return 0;
    for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        cudaSetDevice(sh->ctx->device);
        cudaStreamSynchronize(sh->ctx->stream);
        return 0;
    });
    host_unregister_all(g->ctx); // the application may free its buffers after postrun_graph()
    tb200_context* root = g->ctx;
    destroy_graph(g);
    cudaSetDevice(root->device);
    return 0;
}

int tb200_graph_weight_arena(tb200_graph* g, void** device_ptr, size_t* bytes)
{
    if (!g || !device_ptr || !bytes) return fail(TB200_ERR_INVALID, "bad arguments");
    *device_ptr = g->w_arena, *bytes = g->w_bytes;
    return 0;
}

int tb200_graph_num_launches(tb200_graph* g)
{
    if (!g) return 0;
    int n = g->cur->num_launches;
    for (tb200_graph* sh : g->shards) n += sh->cur->num_launches;
    return n;
}

const char* tb200_graph_layer_kernel(tb200_graph* g, int layer)
{
    if (!g || layer < 0 || layer >= (int)g->layer_kernel.size()) return "";
    return g->layer_kernel[layer];
}

int tb200_graph_read_tensor(tb200_graph* g, int tensor_id, void* host_nchw)
{
    if (!g || tensor_id < 0 || tensor_id >= (int)g->tensors.size() || !host_nchw) return fail(TB200_ERR_INVALID, "bad arguments");
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const TensorInfo& t = sh->tensors[tensor_id];
        uint8_t* tmp = nullptr;
        const size_t bytes = active_nchw_bytes(sh, t);
        CUDA_OK(cudaMalloc(&tmp, bytes));
        cudaError_t e = launch_nhwc_to_nchw(t.dev, tmp, active_dim0(sh, t), t.d.dims[1], t.d.dims[2], t.d.dims[3], sh->ctx->stream);
        if (e == cudaSuccess)
            e = host_copy(g->ctx, (uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, tensor_id), tmp, bytes, cudaMemcpyDeviceToHost, sh->ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(sh->ctx->stream);
        cudaFree(tmp);
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "read_tensor: %s", cudaGetErrorString(e));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_profile(tb200_graph* g, float* layer_ms, int num_layers)
{
    if (!g || !layer_ms || num_layers < (int)g->layers.size()) return fail(TB200_ERR_INVALID, "bad arguments");
    CUDA_OK(cudaSetDevice(g->ctx->device)); // the shard of GPU 0 (every shard runs the same launch sequence on its slice)
    for (int i = 0; i < num_layers; i++) layer_ms[i] = 0.f;
    cudaEvent_t a, b;
    CUDA_OK(cudaEventCreate(&a));
    CUDA_OK(cudaEventCreate(&b));
    int rc = 0;
    for (const Step& s : g->cur->steps)
    {
        cudaEventRecord(a, g->ctx->stream);
        rc = run_step(g, s, g->ctx->stream);
        cudaEventRecord(b, g->ctx->stream);
        if (rc) break;
        if (cudaEventSynchronize(b) != cudaSuccess)
        {
            rc = fail(TB200_ERR_CUDA, "profile: %s", cudaGetErrorString(cudaGetLastError()));
            break;
        }
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        if (s.layer >= 0) layer_ms[s.layer] += ms;
    }
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    return rc;
}

// Tables of the per-byte functions of the examples' post-processing, with their own arithmetic: dequantisation
// ((float)q - zp) * scale (tm_yolov3_tiny_uint8.cpp:471-478), sigmoid = (float)(1.f / (1.f + exp(-x))) (:46-49; tm_yolov5s.cpp:50-53
// is the same function), and exp(x) kept in double because `float pred_w = exp(dw) * anchor_w` multiplies before narrowing (:230).
// The YOLOv5 box formula uses only the sigmoid table.
static void build_yolo_tables(const tb200_tensor_desc& d, float* sig, double* ex)
{
    for (int b = 0; b < 256; b++)
    {
        const float q = d.data_type == TB200_DT_UINT8 ? (float)b : (float)(int)(int8_t)b;
        volatile float x = (q - (float)d.zero_point) * d.scale;
        // The example's `exp(-x)` / `exp(dw)` on a float argument resolve to the float overload (its <cmath> / <math.h> put std::exp(float)
        // in scope): float arithmetic throughout -- pinned by compiling the unmodified example (oracle/yolo_example_shim.cpp,
        // tests/test_yolo_post_pinned.py).  The product exp(dw) * anchor is then a float product: held as a double here, the
        // kernel's double multiply of two float values is exact and its narrowing rounds once, like the float multiply.
        volatile float e_neg = expf(-x), e_pos = expf(x);
        sig[b] = 1.f / (1.f + e_neg);
        ex[b] = (double)e_pos;
    }
}

// Shared by tb200_graph_yolo_detect and tb200_graph_yolov5_detect: the formula only picks the decode kernel's box arithmetic.
static int yolo_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts, YoloBox f)
{
    if (!g || !p || !out || !counts || max_per_image < 1 || p->num_heads < 1 || p->num_heads > 3) return fail(TB200_ERR_INVALID, "bad arguments");
    const int max_cand = p->max_candidates > 0 ? p->max_candidates : 4096;
    static_assert(sizeof(YoloDet) == sizeof(tb200_detection), "detection record layout");
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        const TensorInfo* heads[3] = {};
        for (int hd = 0; hd < p->num_heads; hd++)
        {
            const tb200_yolo_head& H = p->heads[hd];
            if (H.output_index < 0 || H.output_index >= (int)sh->output_ids.size())
                return fail(TB200_ERR_INVALID, "yolo head %d: output index %d", hd, H.output_index);
            heads[hd] = &sh->tensors[sh->output_ids[H.output_index]];
            if (heads[hd]->d.dims[1] != 3 * (p->num_classes + 5))
                return fail(TB200_ERR_INVALID, "yolo head %d: %d channels, expected 3 x (5 + %d)", hd, heads[hd]->d.dims[1], p->num_classes);
        }
        // every head's tables in one block, uploaded by one copy; it stays alive until the stream is synchronised below
        struct YoloTables
        {
            double ex[3][256];
            float sig[3][256];
        } tab;
        for (int hd = 0; hd < p->num_heads; hd++) build_yolo_tables(heads[hd]->d, tab.sig[hd], tab.ex[hd]);
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        cudaGetLastError(); // the launches below report cudaGetLastError(): a non-sticky error an earlier call left behind is not theirs
        cudaStream_t st = sh->ctx->stream;
        const int n_img = sh->num_images;
        YoloCand *cand = nullptr, *sorted = nullptr;
        YoloDet* det = nullptr;
        int *cnt = nullptr, *ocnt = nullptr;
        uint8_t* dtab = nullptr;
        auto cleanup = [&]() { cudaFree(cand), cudaFree(sorted), cudaFree(det), cudaFree(cnt), cudaFree(ocnt), cudaFree(dtab); };
        cudaError_t e = cudaMalloc(&cand, sizeof(YoloCand) * (size_t)n_img * max_cand);
        if (e == cudaSuccess) e = cudaMalloc(&sorted, sizeof(YoloCand) * (size_t)n_img * max_cand);
        if (e == cudaSuccess) e = cudaMalloc(&det, sizeof(YoloDet) * (size_t)n_img * max_per_image);
        if (e == cudaSuccess) e = cudaMalloc(&cnt, sizeof(int) * n_img);
        if (e == cudaSuccess) e = cudaMalloc(&ocnt, sizeof(int) * n_img);
        if (e == cudaSuccess) e = cudaMalloc(&dtab, sizeof tab);
        if (e == cudaSuccess) e = cudaMemsetAsync(cnt, 0, sizeof(int) * n_img, st);
        if (e == cudaSuccess) e = host_copy(g->ctx, dtab, &tab, sizeof tab, cudaMemcpyHostToDevice, st);
        const double* ex = (const double*)dtab;
        const float* sig = (const float*)(dtab + offsetof(YoloTables, sig));
        unsigned key_base = 0;
        for (int hd = 0; hd < p->num_heads && e == cudaSuccess; hd++)
        {
            const TensorInfo& t = *heads[hd];
            const tb200_yolo_head& H = p->heads[hd];
            e = launch_yolo_decode(f, t.dev, t.cp, t.d.dims[2], t.d.dims[3], n_img, p->num_classes, sig + hd * 256, ex + hd * 256, (float)H.stride, H.anchors,
                                   p->prob_threshold, cand, cnt, max_cand, key_base, t.d.data_type == TB200_DT_UINT8, st);
            key_base += (unsigned)(t.d.dims[2] * t.d.dims[3] * 3);
        }
        if (e == cudaSuccess) e = launch_yolo_nms(cand, cnt, n_img, max_cand, p->nms_threshold, sorted, det, max_per_image, ocnt, st);
        if (e == cudaSuccess)
            e = host_copy(g->ctx, out + (size_t)sh->first_image * max_per_image, det, sizeof(YoloDet) * (size_t)n_img * max_per_image, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = host_copy(g->ctx, counts + sh->first_image, ocnt, sizeof(int) * n_img, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cleanup();
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "yolo_detect: %s", cudaGetErrorString(e));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_yolo_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts)
{
    return yolo_detect(g, p, out, max_per_image, counts, YoloBox::V3);
}

int tb200_graph_yolov5_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts)
{
    return yolo_detect(g, p, out, max_per_image, counts, YoloBox::V5);
}

// The argument checks tb200_graph_topk and tb200k_class_topk share; 0 when the launch may go ahead.
static int class_topk_check(int data_type, float scale, long long e, int k)
{
    static_assert(CLASS_TOPK_MAX_K == TB200_TOPK_MAX && CLASS_TOPK_MAX_CLASSES == TB200_TOPK_MAX_CLASSES, "top-k limits");
    static_assert(sizeof(ClassScore) == sizeof(tb200_class_score) && offsetof(ClassScore, id) == offsetof(tb200_class_score, id), "class score record layout");
    if (data_type != TB200_DT_INT8 && data_type != TB200_DT_UINT8) return fail(TB200_ERR_INVALID, "topk: data type %d is not int8 / uint8", data_type);
    if (k < 1 || k > TB200_TOPK_MAX) return fail(TB200_ERR_INVALID, "topk: k = %d outside 1..%d", k, TB200_TOPK_MAX);
    if (k > e) return fail(TB200_ERR_INVALID, "topk: k = %d of %lld classes", k, e);
    // a NaN score fails both of sort_cls_score's comparisons, so neither scan moves and the example's loop never ends: there is no
    // result to reproduce.  A finite scale cannot produce one (scores are finite or infinite, which compare like any number).
    if (!std::isfinite(scale)) return fail(TB200_ERR_INVALID, "topk: scale %g is not finite", (double)scale);
    if (e > TB200_TOPK_MAX_CLASSES) return fail(TB200_ERR_UNSUPPORTED, "topk: %lld classes per image, at most %d are staged", e, TB200_TOPK_MAX_CLASSES);
    return 0;
}

int tb200_graph_topk(tb200_graph* g, int output_index, int k, tb200_class_score* out)
{
    if (!g || !out || output_index < 0 || output_index >= (int)g->output_ids.size()) return fail(TB200_ERR_INVALID, "bad topk arguments");
    {
        const tb200_tensor_desc& d = g->tensors[g->output_ids[output_index]].d;
        if (const int rc = class_topk_check(d.data_type, d.scale, (long long)d.dims[1] * d.dims[2] * d.dims[3], k)) return rc;
    }
    const int rc = for_each_busy_shard(g, [&](tb200_graph* sh, int) -> int {
        const TensorInfo& t = sh->tensors[sh->output_ids[output_index]];
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        cudaGetLastError(); // the launch below reports cudaGetLastError(): a non-sticky error an earlier call left behind is not its own
        cudaStream_t st = sh->ctx->stream;
        const size_t bytes = sizeof(ClassScore) * (size_t)sh->num_images * k;
        ClassScore* dev = nullptr;
        cudaError_t e = cudaMalloc(&dev, bytes);
        if (e == cudaSuccess)
            e = launch_class_topk(t.dev, sh->num_images, t.d.dims[1], t.d.dims[2], t.d.dims[3], t.d.data_type == TB200_DT_UINT8, t.d.scale, t.d.zero_point, k, dev, st);
        if (e == cudaSuccess) e = host_copy(g->ctx, out + (size_t)sh->first_image * k, dev, bytes, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cudaFree(dev);
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "topk: %s", cudaGetErrorString(e));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_work(tb200_graph* g, double* ops, double* bytes)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    double o = g->cur->work_ops, b = g->cur->work_bytes;
    for (tb200_graph* sh : g->shards) o += sh->cur->work_ops, b += sh->cur->work_bytes - sh->cur->work_wbytes; // weights count once per launch
    if (ops) *ops = o;
    if (bytes) *bytes = b;
    return 0;
}

// ---- kernel-level entry points (device pointers) -------------------------------------------------------------
static EpiParams epi_from_abi(const tb200k_epilogue* e)
{
    EpiParams p{};
    p.bias = e->bias, p.w_scale = e->w_scale, p.in_scale = e->in_scale, p.out_scale = e->out_scale;
    p.in_zero = e->in_zero, p.w_zero = e->w_zero, p.out_zero = e->out_zero, p.activation = e->activation, p.recipe = e->recipe;
    p.is_uint8 = e->is_uint8, p.fc_rounding = e->fc_rounding, p.has_bias = e->bias != nullptr;
    p.in_w_scale = e->in_scale * e->w_scale_tensor;
    p.bias_scale = p.in_w_scale;
    p.fast_ok = 0; // the raw kernel entry points always use the literal reference arithmetic
    return p;
}
static ConvShape shape_from_abi(const tb200k_conv_shape* s)
{
    ConvShape c{};
    c.n = s->n, c.h = s->h, c.w = s->w, c.c = s->c, c.cp = cpad(s->c), c.oh = s->oh, c.ow = s->ow, c.oc = s->oc, c.ocp = cpad(s->oc);
    c.kh = s->kh, c.kw = s->kw, c.sh = s->sh, c.sw = s->sw, c.ph0 = s->ph0, c.pw0 = s->pw0, c.dh = s->dh, c.dw = s->dw, c.group = s->group;
    c.cg = s->c / s->group, c.cgp = s->group == 1 ? c.cp : c.cg;
    return c;
}
#define K_CHECK(cond) \
    if (!(cond)) return fail(TB200_ERR_INVALID, "invalid kernel arguments: %s", #cond)
#define K_LAUNCH(expr)                                                                      \
    do                                                                                      \
    {                                                                                       \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) return fail(TB200_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
        return 0;                                                                           \
    } while (0)

int tb200k_conv_direct(const void* in, const void* weight, void* out, const tb200k_conv_shape* s, const tb200k_epilogue* e, void* stream)
{
    K_CHECK(in && weight && out && s && e && s->group >= 1);
    EpiParams p = epi_from_abi(e);
    K_LAUNCH(launch_conv_direct(in, weight, out, shape_from_abi(s), p, (cudaStream_t)stream));
}
int tb200k_conv_dw3x3(const void* in, const void* weight, void* out, const tb200k_conv_shape* s, const tb200k_epilogue* e, void* stream)
{
    K_CHECK(in && weight && out && s && e && s->group == s->c && s->oc == s->c);
    EpiParams p = epi_from_abi(e);
    K_LAUNCH(launch_conv_dw(in, weight, out, shape_from_abi(s), p, (cudaStream_t)stream));
}
int tb200k_conv_stem_nchw(const void* in_nchw, const void* weight, void* out, const tb200k_conv_shape* s, const tb200k_epilogue* e, void* stream)
{
    K_CHECK(in_nchw && weight && out && s && e && s->c <= 4 && s->group == 1);
    EpiParams p = epi_from_abi(e);
    K_LAUNCH(launch_conv_stem(in_nchw, weight, out, shape_from_abi(s), p, (cudaStream_t)stream));
}
int tb200k_gemm_i8(const void* in, const void* weight, void* out, int64_t m, int32_t k_pad, int32_t oc, const tb200k_epilogue* e, void* stream)
{
    K_CHECK(in && weight && out && e && m > 0 && k_pad > 0 && oc > 0 && !e->is_uint8);
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return fail(TB200_ERR_NO_DEVICE, "no CUDA device");
    GemmPlan plan;
    int rc = gemm_plan_create(&plan, in, k_pad, weight, out, m, k_pad, oc, cpad(oc), cpad(oc), 0);
    if (rc) return fail(rc, "gemm plan failed");
    EpiParams p = epi_from_abi(e);
    K_LAUNCH(launch_gemm_i8(plan, p, nullptr, sms, (cudaStream_t)stream));
}
size_t tb200k_conv_winograd43_f32_workspace(const tb200k_conv_shape* s) { return s ? wino43_workspace_bytes(s->n, s->c, s->oc, s->oh, s->ow) : 0; }
int tb200k_conv_winograd43_f32(const float* in, const float* weight, const float* bias, float* out, const tb200k_conv_shape* s, int activation, void* workspace,
                               void* stream)
{
    K_CHECK(in && weight && out && s && workspace && s->kh == 3 && s->kw == 3 && s->sh == 1 && s->sw == 1 && s->dh == 1 && s->dw == 1 && s->group == 1);
    K_CHECK(s->oh == s->h + 2 * s->ph0 - 2 && s->ow == s->w + 2 * s->pw0 - 2);
    K_LAUNCH(launch_conv_winograd43_f32(in, weight, bias, out, s->n, s->c, s->h, s->w, s->oc, s->oh, s->ow, s->ph0, s->pw0, activation, (float*)workspace,
                                        (cudaStream_t)stream));
}
int tb200k_conv_dw3x3_f32(const float* in, const float* weight, const float* bias, float* out, const tb200k_conv_shape* s, int activation, void* stream)
{
    K_CHECK(in && weight && out && s && s->kh == 3 && s->kw == 3 && s->sh == s->sw && (s->sh == 1 || s->sh == 2) && s->dh == 1 && s->dw == 1 &&
            s->group == s->c && s->oc == s->c);
    K_LAUNCH(launch_conv_dw3x3_f32(in, weight, bias, out, s->n, s->c, s->h, s->w, s->oh, s->ow, s->sh, s->ph0, s->pw0, activation, (cudaStream_t)stream));
}
int tb200k_nchw_to_nhwc(const void* in, void* out, int n, int c, int h, int w, void* stream)
{
    K_CHECK(in && out && n > 0 && c > 0 && h > 0 && w > 0);
    K_LAUNCH(launch_nchw_to_nhwc(in, out, n, c, h, w, (cudaStream_t)stream));
}
int tb200k_nhwc_to_nchw(const void* in, void* out, int n, int c, int h, int w, void* stream)
{
    K_CHECK(in && out && n > 0 && c > 0 && h > 0 && w > 0);
    K_LAUNCH(launch_nhwc_to_nchw(in, out, n, c, h, w, (cudaStream_t)stream));
}

int tb200k_class_topk(const void* in, int n, int c, int h, int w, int is_uint8, float scale, int32_t zero_point, int k, tb200_class_score* out, void* stream)
{
    K_CHECK(in && out && n > 0 && c > 0 && h > 0 && w > 0);
    if (const int rc = class_topk_check(is_uint8 ? TB200_DT_UINT8 : TB200_DT_INT8, scale, (long long)c * h * w, k)) return rc;
    K_LAUNCH(launch_class_topk(in, n, c, h, w, is_uint8 != 0, scale, zero_point, k, (ClassScore*)out, (cudaStream_t)stream));
}
} // extern "C"
