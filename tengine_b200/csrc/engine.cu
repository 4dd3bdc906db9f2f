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
#define TB200_PACK_FORMAT 4  // bump whenever the layout or content of the packed weight arena changes (pack cache key)

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
    K_STEM_TC,
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
static const char* kStepName[] = {"nchw_to_nhwc", "nhwc_to_nchw", "conv_stem_nchw_dp4a", "conv_stem_nchw_tcgen05", "conv_gather_tcgen05", "conv_dw_direct", "conv_direct_dp4a",
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

struct tb200_graph
{
    tb200_context* ctx;
    int flags;
    std::vector<TensorInfo> tensors;
    std::vector<tb200_layer_desc> layers;
    std::vector<const char*> layer_kernel;
    std::vector<Step> steps;
    std::vector<int> input_ids, output_ids;
    std::vector<uint8_t*> in_nchw_dev, out_nchw_dev;
    uint8_t* act_arena = nullptr;
    size_t act_bytes = 0;
    uint8_t* w_arena = nullptr;
    size_t w_bytes = 0;
    int chunks = 1;
    std::vector<int> chunk_first, chunk_count; // images of pipeline chunk k: [first, first + count)
    std::vector<std::vector<Step>> chunk_steps;
    std::vector<cudaGraph_t> cu_graphs;
    std::vector<cudaGraphExec_t> cu_execs;
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_out;
    cudaEvent_t ev_done = nullptr;
    double work_ops = 0, work_bytes = 0, work_wbytes = 0;
    int num_launches = 0;
    // batch sharding over the GPUs of a multi-GPU context: this graph is the shard of GPU 0 and owns the others
    std::vector<tb200_graph*> shards;
    int first_image = 0, num_images = 0, total_images = 0;
    size_t act_unshared_bytes = 0; // what the arena would need without slot reuse (introspection)
    int pack_cache_state = 0;      // 0 no cache directory, 1 packed and written, 2 read from the cache
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

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
    static const bool no_fixq = getenv("TB200_NO_FIXQ") != nullptr; // A/B switch: guarded elements fixed inline
    if (!no_fixq) CUDA_OK(cudaMalloc(&c->fixq, (size_t)sms * FIXQ_CAP * 16));
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
        // integer-domain clip + zero point + saturation (common.cuh requant_fast8_u8): the activation bounds become the integers
        // the reference's own division and round() give for them; q' = max(min(q + zp - L, H - L), 0), byte = q' + L
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

// bytes of the packed B operand of the tensor-core paths: [n_tiles][block_n (+16 for uint8: the ones-row)][K]
static size_t gemm_weight_bytes(int ocp, int k, bool u8)
{
    const int bn = gemm_block_n(ocp, u8), nt = (ocp + bn - 1) / bn;
    return (size_t)nt * (bn + (u8 ? 16 : 0)) * k;
}

struct WeightBlob
{
    size_t w_off, bias_off, scale_off, fast_off, btab_off, w_size;
};

static int run_step(tb200_graph* g, const Step& s, cudaStream_t st)
{
    cudaError_t err = cudaSuccess;
    switch (s.kind)
    {
    case K_NCHW2NHWC: err = launch_nchw_to_nhwc(s.in, s.out, s.n, s.c, s.h, s.w_, st); break;
    case K_NHWC2NCHW: err = launch_nhwc_to_nchw(s.in, s.out, s.n, s.c, s.h, s.w_, st); break;
    case K_CONV_STEM: err = launch_conv_stem(s.in, s.w, s.out, s.cs, s.epi, st); break;
    case K_STEM_TC: err = launch_stem_tc(s.dwp, s.in, s.w, s.out, s.cs, s.epi, st); break;
    case K_GATHER_TC:
        err = s.wp.valid ? launch_conv_window(s.wp, s.w, s.out, s.cs, s.epi, st) : launch_conv_gather_tc(s.in, s.w, s.out, s.cs, s.epi, s.nhwc16, st);
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

static void destroy_graph(tb200_graph* g)
{
    if (!g) return;
    for (tb200_graph* sh : g->shards) destroy_graph(sh);
    g->shards.clear();
    cudaSetDevice(g->ctx->device);
    for (auto e : g->cu_execs) if (e) cudaGraphExecDestroy(e);
    for (auto c : g->cu_graphs) if (c) cudaGraphDestroy(c);
    for (auto e : g->ev_in) cudaEventDestroy(e);
    for (auto e : g->ev_out) cudaEventDestroy(e);
    if (g->ev_done) cudaEventDestroy(g->ev_done);
    if (g->copy_stream) cudaStreamDestroy(g->copy_stream);
    if (g->d2h_stream) cudaStreamDestroy(g->d2h_stream);
    for (auto p : g->in_nchw_dev) cudaFree(p);
    for (auto p : g->out_nchw_dev) cudaFree(p);
    cudaFree(g->act_arena);
    cudaFree(g->w_arena);
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

static int prerun_one(tb200_context* ctx, const tb200_tensor_desc* tensors, int num_tensors, const tb200_layer_desc* layers, int num_layers,
                      const int32_t* input_ids, int num_inputs, const int32_t* output_ids, int num_outputs, int flags, tb200_graph* g)
{
    CUDA_OK(cudaSetDevice(ctx->device));
    auto bail = [&](int rc) { return rc; }; // the caller owns g and destroys it on failure (arenas, tensor maps, CUDA graphs, an open capture)

    // ---- node fusion (SURVEY.md 8(f)-1), decided from the descriptors alone.  Eltwise -> ReLU where the ReLU's output has its
    //      input's quantisation (what the reference's quantisation tool writes, quant_save_graph.cpp:136-200) and the eltwise
    //      result has no other reader: the ReLU is then max(byte, zero point) on the requantised bytes (relu_same_scale_kernel),
    //      applied inside the eltwise kernel -- one pass over memory instead of two, the intermediate tensor is never stored.
    //      Not under TB200_PRERUN_NO_GRAPH, whose contract is that every intermediate stays readable. ----
    const std::vector<tb200_layer_desc> src_layers(layers, layers + num_layers); // the descriptors as the caller gave them
    std::vector<tb200_layer_desc> fused(layers, layers + num_layers);
    std::vector<int> post_relu(num_layers, 0);
    if (!(flags & TB200_PRERUN_NO_GRAPH) && !getenv("TB200_NO_FUSION"))
    {
        std::vector<int> readers(num_tensors, 0), reader_layer(num_tensors, -1);
        for (int li = 0; li < num_layers; li++)
            for (int k = 0; k < layers[li].num_inputs && k < 4; k++)
                if (layers[li].inputs[k] >= 0 && layers[li].inputs[k] < num_tensors) readers[layers[li].inputs[k]]++, reader_layer[layers[li].inputs[k]] = li;
        std::vector<char> is_out(num_tensors, 0);
        for (int i = 0; i < num_outputs; i++)
            if (output_ids[i] >= 0 && output_ids[i] < num_tensors) is_out[output_ids[i]] = 1;
        for (int li = 0; li < num_layers; li++)
        {
            const tb200_layer_desc& E = layers[li];
            if (E.op != TB200_OP_ELTWISE || E.output < 0 || E.output >= num_tensors || readers[E.output] != 1 || is_out[E.output]) continue;
            const int lj = reader_layer[E.output];
            const tb200_layer_desc& R = layers[lj];
            if (lj <= li || R.op != TB200_OP_RELU || R.negative_slope != 0.f || R.output < 0 || R.output >= num_tensors) continue;
            const tb200_tensor_desc &ti = tensors[E.output], &to = tensors[R.output];
            if (ti.scale != to.scale || ti.zero_point != to.zero_point || ti.data_type != to.data_type) continue;
            if (ti.data_type == TB200_DT_UINT8 && (ti.dims[1] % 16)) continue; // pad lanes of uint8 tensors must stay 0, not the zero point
            bool same = true;
            for (int k = 0; k < 4; k++) same &= ti.dims[k] == to.dims[k];
            if (!same) continue;
            fused[li].output = R.output, post_relu[li] = 1;
            fused[lj].op = TB200_OP_NOP_, fused[lj].num_inputs = 0;
        }
    }
    // (Leaky) ReLU -> max pooling whose output keeps the ReLU's quantisation, the ReLU result having no other reader: the ReLU is
    // a non-decreasing byte table, so max(table(x)) == table(max(x)); the pooling reads the convolution's bytes and applies the
    // table to each window's maximum.  One pass over the big tensor disappears (pool_relu[pool layer] = the folded ReLU layer).
    std::vector<int> pool_relu(num_layers, -1);
    if (!(flags & TB200_PRERUN_NO_GRAPH) && !getenv("TB200_NO_FUSION"))
    {
        std::vector<int> readers(num_tensors, 0), reader_layer(num_tensors, -1);
        for (int li = 0; li < num_layers; li++)
            for (int k = 0; k < fused[li].num_inputs && k < 4; k++)
                if (fused[li].inputs[k] >= 0 && fused[li].inputs[k] < num_tensors) readers[fused[li].inputs[k]]++, reader_layer[fused[li].inputs[k]] = li;
        std::vector<char> is_out(num_tensors, 0);
        for (int i = 0; i < num_outputs; i++)
            if (output_ids[i] >= 0 && output_ids[i] < num_tensors) is_out[output_ids[i]] = 1;
        for (int li = 0; li < num_layers; li++)
        {
            const tb200_layer_desc& R = fused[li];
            if (R.op != TB200_OP_RELU || R.output < 0 || R.output >= num_tensors || readers[R.output] != 1 || is_out[R.output]) continue;
            if (!(R.negative_slope >= 0.f && R.negative_slope <= 1.f)) continue; // the table must be non-decreasing
            const int lj = reader_layer[R.output];
            const tb200_layer_desc& P = fused[lj];
            if (lj <= li || P.op != TB200_OP_POOL || P.pool_method != TB200_POOL_MAX || P.output < 0 || P.output >= num_tensors) continue;
            const tb200_tensor_desc &tr = tensors[R.output], &tp = tensors[P.output];
            if (tr.scale != tp.scale || tr.zero_point != tp.zero_point || tr.data_type != tp.data_type) continue;
            pool_relu[lj] = li;
            fused[lj].inputs[0] = R.inputs[0]; // the pooling reads what the ReLU read
            fused[li].op = TB200_OP_NOP_, fused[li].num_inputs = 0;
        }
    }
    // Sigmoid -> Eltwise-PROD with the Sigmoid's own input (x * sigmoid(x): how an int8 YOLOv5s spells SiLU, SURVEY.md 8(a)): both
    // operands of the product are functions of the same byte of x, so the PAIR is one byte table -- sigmoid's table composed with
    // the reference's eltwise arithmetic, built at prerun -- and one pass (1 read, 1 write) replaces two (3 reads, 2 writes).
    std::vector<int> silu_sig(num_layers, -1); // [eltwise layer] = the folded Sigmoid layer
    if (!(flags & TB200_PRERUN_NO_GRAPH) && !getenv("TB200_NO_FUSION"))
    {
        std::vector<int> readers(num_tensors, 0), reader_layer(num_tensors, -1);
        for (int li = 0; li < num_layers; li++)
            for (int k = 0; k < fused[li].num_inputs && k < 4; k++)
                if (fused[li].inputs[k] >= 0 && fused[li].inputs[k] < num_tensors) readers[fused[li].inputs[k]]++, reader_layer[fused[li].inputs[k]] = li;
        std::vector<char> is_out(num_tensors, 0);
        for (int i = 0; i < num_outputs; i++)
            if (output_ids[i] >= 0 && output_ids[i] < num_tensors) is_out[output_ids[i]] = 1;
        for (int li = 0; li < num_layers; li++)
        {
            const tb200_layer_desc& S = fused[li];
            if (S.op != TB200_OP_SIGMOID || S.output < 0 || S.output >= num_tensors || readers[S.output] != 1 || is_out[S.output]) continue;
            const int lj = reader_layer[S.output];
            const tb200_layer_desc& E = fused[lj];
            if (lj <= li || E.op != TB200_OP_ELTWISE || E.elt_type != TB200_ELT_PROD || E.num_inputs != 2 || post_relu[lj]) continue;
            const int other = E.inputs[0] == S.output ? E.inputs[1] : (E.inputs[1] == S.output ? E.inputs[0] : -1);
            if (other != S.inputs[0]) continue;
            silu_sig[lj] = li;
            fused[lj].op = TB200_OP_LUT2_, fused[lj].num_inputs = 1, fused[lj].inputs[0] = S.inputs[0];
            fused[lj].axis = (E.inputs[0] == S.output) ? 0 : 1; // which operand of the product was the sigmoid (operand scales differ)
            fused[li].op = TB200_OP_NOP_, fused[li].num_inputs = 0;
        }
    }
    layers = fused.data();

    // ---- tensors ----
    g->tensors.resize(num_tensors);
    size_t act = 0;
    for (int i = 0; i < num_tensors; i++)
    {
        TensorInfo& t = g->tensors[i];
        t.d = tensors[i];
        if (t.d.data_type != TB200_DT_INT8 && t.d.data_type != TB200_DT_UINT8)
            return bail(fail(TB200_ERR_UNSUPPORTED, "tensor %d: data type %d not supported by the H100 backend", i, t.d.data_type));
        for (int k = 0; k < 4; k++)
            if (t.d.dims[k] <= 0) return bail(fail(TB200_ERR_INVALID, "tensor %d: dim %d is %d", i, k, t.d.dims[k]));
        t.cp = cpad(t.d.dims[1]);
        t.nhwc_bytes = (size_t)t.d.dims[0] * t.d.dims[2] * t.d.dims[3] * t.cp;
        t.nchw_bytes = (size_t)t.d.dims[0] * t.d.dims[1] * t.d.dims[2] * t.d.dims[3];
        t.off = 0;
        t.slot_bytes = align_up(t.nhwc_bytes, 1024);
    }
    for (int i = 0; i < num_inputs; i++)
    {
        if (input_ids[i] < 0 || input_ids[i] >= num_tensors) return bail(fail(TB200_ERR_INVALID, "input id out of range"));
        g->tensors[input_ids[i]].input_index = i;
        g->input_ids.push_back(input_ids[i]);
    }
    for (int i = 0; i < num_outputs; i++)
    {
        if (output_ids[i] < 0 || output_ids[i] >= num_tensors) return bail(fail(TB200_ERR_INVALID, "output id out of range"));
        g->tensors[output_ids[i]].output_index = i;
        g->output_ids.push_back(output_ids[i]);
    }
    g->layers.assign(layers, layers + num_layers);
    g->layer_kernel.assign(num_layers, "");

    // ---- validate layers, decide kernels, size the weight arena ----
    std::vector<int> kind(num_layers, -1);
    std::vector<WeightBlob> blobs(num_layers);
    std::vector<int> fuse_bias(num_layers, 0);
    size_t wtotal = 0;
    const bool no_tc = (flags & TB200_PRERUN_NO_TENSORCORE) != 0;
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = layers[li];
        if (L.op == TB200_OP_NOP_)
        {
            kind[li] = K_NONE;
            continue;
        }
        if (L.num_inputs < 1 || L.num_inputs > 4) return bail(fail(TB200_ERR_INVALID, "layer %d: num_inputs %d", li, L.num_inputs));
        for (int k = 0; k < L.num_inputs; k++)
            if (L.inputs[k] < 0 || L.inputs[k] >= num_tensors) return bail(fail(TB200_ERR_INVALID, "layer %d: input id", li));
        if (L.output < 0 || L.output >= num_tensors) return bail(fail(TB200_ERR_INVALID, "layer %d: output id", li));
        TensorInfo& tin = g->tensors[L.inputs[0]];
        TensorInfo& tout = g->tensors[L.output];
        tout.producer = li;
        if (tin.d.data_type != tout.d.data_type) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: mixed data types", li));
        const bool u8 = tin.d.data_type == TB200_DT_UINT8;
        const int C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3], OC = tout.d.dims[1];
        if (L.op == TB200_OP_CONV)
        {
            if (!L.weight || !L.weight_scales) return bail(fail(TB200_ERR_INVALID, "layer %d: conv without weight/scales", li));
            if (L.group < 1 || C % L.group || OC % L.group) return bail(fail(TB200_ERR_INVALID, "layer %d: bad group %d", li, L.group));
            const int oh = (H + L.pad_h0 + L.pad_h1 - (L.dilation_h * (L.kernel_h - 1) + 1)) / L.stride_h + 1;
            const int ow = (W + L.pad_w0 + L.pad_w1 - (L.dilation_w * (L.kernel_w - 1) + 1)) / L.stride_w + 1;
            if (oh != tout.d.dims[2] || ow != tout.d.dims[3] || tout.d.dims[0] != tin.d.dims[0])
                return bail(fail(TB200_ERR_INVALID, "layer %d: conv output shape %dx%d does not match descriptor %dx%d", li, oh, ow, tout.d.dims[2], tout.d.dims[3]));
            const int cg = C / L.group;
            size_t wsize;
            if (tin.input_index >= 0 && C <= 3 && L.group == 1 && !u8 && !no_tc && L.kernel_h == 3 && L.kernel_w == 3 && L.dilation_h == 1 &&
                L.dilation_w == 1 && L.stride_h == L.stride_w && tout.cp <= 256 && !getenv("TB200_NO_STEM_TC"))
                kind[li] = K_STEM_TC, wsize = (size_t)tout.cp * 32; // one 32-byte wgmma k-step per output channel
            else if (tin.input_index >= 0 && C <= 3 && L.group == 1 && !no_tc && L.kernel_h == L.kernel_w && (L.kernel_h == 7 || (u8 && L.kernel_h == 3)) &&
                     L.dilation_h == 1 && L.dilation_w == 1 && L.stride_h == L.stride_w && tout.cp <= 256 && !getenv("TB200_NO_GATHER_TC"))
                // uint8 3x3 stems and 7x7 stems (ResNet): threads gather, taps outside the image = zero point; K padded to 32*ks
                kind[li] = K_GATHER_TC, wsize = (size_t)tout.cp * 32 * ((C * L.kernel_h * L.kernel_w + 31) / 32);
            else if (tin.input_index >= 0 && C <= 4 && L.group == 1)
                kind[li] = K_CONV_STEM, wsize = (size_t)tout.cp * L.kernel_h * L.kernel_w * 4;
            else if (!no_tc && L.group == 1 && tin.cp == 16 && L.kernel_h == 3 && L.kernel_w == 3 && L.dilation_h == 1 && L.dilation_w == 1 &&
                     L.stride_h == L.stride_w && tout.cp <= 256 && !getenv("TB200_NO_GATHER_TC"))
                kind[li] = K_GATHER_TC, wsize = (size_t)tout.cp * 160; // 16-channel input: nine 16-byte taps per pixel, five k-steps
            else if (!no_tc && L.group == 1 && tin.cp == 32 && L.kernel_h == 3 && L.kernel_w == 3 && L.dilation_h == 1 &&
                     L.dilation_w == 1 && L.stride_h == L.stride_w && (L.stride_h == 1 || L.stride_h == 2) && tout.cp <= 256 &&
                     window_nhwc_fits(32, tout.cp, L.stride_h) && !getenv("TB200_NO_GATHER_TC") && !getenv("TB200_NO_WINDOW_CONV"))
                kind[li] = K_GATHER_TC, wsize = (size_t)tout.cp * 288; // 32-channel input through the window kernel: nine 32-byte taps = nine k-steps
            else if (L.group == C && OC == C && C > 1)
                kind[li] = K_CONV_DW, wsize = (size_t)L.kernel_h * L.kernel_w * tin.cp;
            else if (!no_tc && L.group == 1 && L.kernel_h == 1 && L.kernel_w == 1 && L.stride_h == 1 && L.stride_w == 1 &&
                     !L.pad_h0 && !L.pad_h1 && !L.pad_w0 && !L.pad_w1 && !(u8 && getenv("TB200_NO_U8_TC")))
                kind[li] = K_GEMM, wsize = gemm_weight_bytes(tout.cp, tin.cp, u8);
            else if (!no_tc && L.group == 1 && L.dilation_h == 1 && L.dilation_w == 1 && L.stride_h == L.stride_w &&
                     (L.stride_h == 1 || L.stride_h == 2) && (L.kernel_h * L.kernel_w == 1 || tin.cp % 32 == 0) && tout.d.dims[3] <= 4096 &&
                     L.kernel_h * L.kernel_w <= 64 && !getenv("TB200_NO_IGEMM") && !(u8 && getenv("TB200_NO_U8_TC")))
                kind[li] = K_IGEMM, wsize = gemm_weight_bytes(tout.cp, L.kernel_h * L.kernel_w * tin.cp, u8);
            else
            {
                if (L.group > 1 && ((cg % 4) || ((OC / L.group) % 4)))
                    return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: grouped conv needs channels per group %% 4 == 0", li));
                kind[li] = K_CONV_DIRECT;
                wsize = (size_t)tout.cp * L.kernel_h * L.kernel_w * (L.group == 1 ? tin.cp : cg);
            }
            blobs[li].w_size = wsize;
        }
        else if (L.op == TB200_OP_FC)
        {
            if (!L.weight || !L.weight_scales) return bail(fail(TB200_ERR_INVALID, "layer %d: fc without weight/scales", li));
            if (no_tc || (u8 && getenv("TB200_NO_U8_TC")))
                kind[li] = K_CONV_DIRECT, blobs[li].w_size = (size_t)tout.cp * H * W * tin.cp; // FC == conv with kernel HxW over the whole input
            else
                kind[li] = K_GEMM, blobs[li].w_size = gemm_weight_bytes(tout.cp, H * W * tin.cp, u8);
        }
        else if (L.op == TB200_OP_POOL)
            kind[li] = K_POOL;
        else if (L.op == TB200_OP_RELU)
            kind[li] = K_POINTWISE;
        else if (L.op == TB200_OP_ELTWISE)
        {
            if (L.num_inputs != 2 || (L.elt_type != TB200_ELT_SUM && L.elt_type != TB200_ELT_PROD))
                return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: eltwise type %d / %d inputs", li, L.elt_type, L.num_inputs));
            kind[li] = K_POINTWISE;
        }
        else if (L.op == TB200_OP_CONCAT)
        {
            if (L.axis != 1) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: concat axis %d", li, L.axis));
            kind[li] = (L.num_inputs == 1) ? K_COPY : K_CONCAT_PART; // concat_kernel_ref_int8.c:45-56: one input is a plain copy
        }
        else if (L.op == TB200_OP_UPSAMPLE)
            kind[li] = K_UPSAMPLE;
        else if (L.op == TB200_OP_IDENTITY)
            kind[li] = K_COPY;
        else if (L.op == TB200_OP_LUT2_)
            kind[li] = K_LUT;
        else if (L.op == TB200_OP_SIGMOID || L.op == TB200_OP_HARDSWISH)
        {
            // the reference has no int8 hardswish (hardswish_ref.c:59-66): nothing to be identical to
            if (L.op == TB200_OP_HARDSWISH && !u8) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: int8 hardswish has no reference kernel", li));
            kind[li] = K_LUT;
        }
        else if (L.op == TB200_OP_SOFTMAX)
        {
            if (L.axis != 1) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: softmax axis %d (only the channel axis)", li, L.axis));
            kind[li] = K_SOFTMAX;
        }
        else if (L.op == TB200_OP_RESHAPE)
        {
            if (tin.nchw_bytes != tout.nchw_bytes || tin.d.dims[0] != tout.d.dims[0])
                return bail(fail(TB200_ERR_INVALID, "layer %d: reshape changes the element count or the batch", li));
            // NHWC(pad) == NCHW order when the tensor is a vector per image or has one channel: a plain copy then
            const bool same = (H * W == 1 && tout.d.dims[2] * tout.d.dims[3] == 1) || (C == tout.d.dims[1] && H == tout.d.dims[2] && W == tout.d.dims[3]);
            kind[li] = same ? K_COPY : K_RESHAPE;
        }
        else
            return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: op %d", li, L.op));

        if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
        {
            blobs[li].w_off = wtotal;
            wtotal += align_up(blobs[li].w_size, 1024);
            blobs[li].bias_off = wtotal;
            wtotal += align_up((size_t)tout.cp * 4, 256);
            blobs[li].scale_off = wtotal;
            wtotal += align_up((size_t)tout.cp * 4, 256);
            blobs[li].fast_off = wtotal;
            wtotal += align_up((size_t)tout.cp * 8, 256);
            blobs[li].btab_off = wtotal;
            if (u8 && kind[li] == K_IGEMM) // [border patterns][OCp] int32, see the packing below
                wtotal += align_up((size_t)(L.pad_h0 + 1) * (L.kernel_h + 1) * (L.pad_w0 + 1) * (L.kernel_w + 1) * tout.cp * 4, 256);
        }
        if (kind[li] == K_LUT || (kind[li] == K_POOL && pool_relu[li] >= 0))
        {
            blobs[li].w_off = wtotal; // 256-byte table; part of the arena so that it travels with the single broadcast
            wtotal += 256;
        }
        if (kind[li] == K_CONCAT_PART)
        {
            blobs[li].w_off = wtotal; // one requantisation table per input
            wtotal += 256 * 4;
        }
        // which graph inputs need an NHWC copy (everything except a stem conv reads NHWC)
        for (int k = 0; k < L.num_inputs; k++)
            if (g->tensors[L.inputs[k]].input_index >= 0 && kind[li] != K_CONV_STEM && kind[li] != K_STEM_TC && !(kind[li] == K_GATHER_TC && g->tensors[L.inputs[k]].d.dims[1] <= 3)) g->tensors[L.inputs[k]].nhwc_needed = true;
    }
    for (int id : g->output_ids)
        if (g->tensors[id].input_index >= 0) g->tensors[id].nhwc_needed = true;

    // ---- activation arena: one 1 KiB-aligned slot per tensor; a slot is handed on once the tensor's last consumer has run
    //      (first-fit over a coalescing free list, the role of source/device/cpu/cpu_pool.c:253-439).  Graph inputs and outputs
    //      keep their slots; with TB200_PRERUN_NO_GRAPH (debug: every intermediate stays readable) nothing is reused. ----
    std::vector<size_t> scratch_off(num_layers, 0);
    {
        const bool reuse = !(flags & TB200_PRERUN_NO_GRAPH) && !getenv("TB200_NO_ARENA_REUSE");
        for (int li = 0; li < num_layers; li++)
            for (int k = 0; k < layers[li].num_inputs; k++) g->tensors[layers[li].inputs[k]].last_use = li;
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
            const tb200_layer_desc& L = layers[li];
            if (L.op == TB200_OP_NOP_) continue;
            TensorInfo& to = g->tensors[L.output];
            if (!placed[L.output]) to.off = alloc(to.slot_bytes), placed[L.output] = 1;
            if (kind[li] == K_RESHAPE)
            {
                const size_t sb = align_up(to.nchw_bytes, 1024);
                scratch_off[li] = alloc(sb);
                g->act_unshared_bytes += sb;
                release(scratch_off[li], sb);
            }
            for (int k = 0; k < L.num_inputs; k++)
            {
                const int id = L.inputs[k];
                TensorInfo& ti = g->tensors[id];
                if (ti.last_use == li && !permanent(ti) && !freed[id]) release(ti.off, ti.slot_bytes), freed[id] = 1;
            }
            if (to.last_use < li && !permanent(to) && !freed[L.output]) release(to.off, to.slot_bytes), freed[L.output] = 1; // dead value
        }
        act = top;
    }
    g->act_bytes = act;
    CUDA_OK(cudaMalloc(&g->act_arena, act ? act : 1024));
    // pad lanes of every tensor are (re)written by its producer; the initial fill only matters for debugging reads
    CUDA_OK(cudaMemsetAsync(g->act_arena, (flags & TB200_PRERUN_POISON_ARENA) ? 0xA5 : 0, act ? act : 1024, ctx->stream));
    for (auto& t : g->tensors) t.dev = g->act_arena + t.off;
    g->w_bytes = wtotal ? wtotal : 1024;
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

    // ---- per layer: may the fast epilogue fold the bias add into its FMA?  (common.cuh requant_fast_bits<.., FUSE>)
    //      Decided from the descriptors alone so that every rank of a sharded job reaches the same arena format. ----
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = layers[li];
        if (L.op != TB200_OP_CONV) continue;
        const TensorInfo& tin = g->tensors[L.inputs[0]];
        const TensorInfo& tout = g->tensors[L.output];
        if (tin.d.data_type == TB200_DT_UINT8 || getenv("TB200_NO_FUSE_BIAS")) continue;
        bool fuse = true;
        for (int o = 0; o < tout.d.dims[1]; o++)
        {
            const double bm = (double)(L.bias ? L.bias[o] : 0) * (double)tin.d.scale * (double)L.weight_scales[o] / (double)tout.d.scale;
            if (!(bm >= -100.0 && bm <= 100.0)) fuse = false;
        }
        fuse_bias[li] = fuse ? 1 : 0;
    }
    // ---- uint8 tensor-core layers use the int8 form of the fast epilogue: t = fl((float)(acc_true + bias) * M), M = fl(s_in*s_w/s_out).
    //      The reference forms f = fl(fl(acc*S) + fl(bias*S)) and t_ref = fl(f / s_out): |t - t_ref| <= 2^-24 (2|bias*M| + 5|t|), which
    //      stays inside the 2^-13 tie guard for every in-range t (|t| <= 255) as long as |bias*M| <= 250 -- checked here per channel;
    //      an FC whose bias tensor carries its own scale (fc_ref.c:141-146) cannot fold the bias into the integer sum at all.
    //      Layers that fail the check take the exact epilogue. ----
    std::vector<int> u8_tc_fast(num_layers, 1);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = layers[li];
        if ((L.op != TB200_OP_CONV && L.op != TB200_OP_FC) || (kind[li] != K_GEMM && kind[li] != K_IGEMM && kind[li] != K_GATHER_TC)) continue;
        const TensorInfo& tin = g->tensors[L.inputs[0]];
        const TensorInfo& tout = g->tensors[L.output];
        if (tin.d.data_type != TB200_DT_UINT8) continue;
        const float S = tin.d.scale * L.weight_scales[0];
        if (L.op == TB200_OP_FC && L.bias && L.bias_scale != 0.f && L.bias_scale != S) u8_tc_fast[li] = 0;
        const double M = (double)tin.d.scale * (double)L.weight_scales[0] / (double)tout.d.scale;
        for (int o = 0; o < tout.d.dims[1] && L.bias; o++)
            if (!(fabs((double)L.bias[o] * M) <= 250.0)) u8_tc_fast[li] = 0;
    }
    // ---- int8 fast epilogue rounds BEFORE it clamps (integer-domain clamp on 16-bit lanes, common.cuh): prove from the
    //      weights that no reachable accumulator can leave the 16-bit range after scaling, else use the exact path ----
    std::vector<int> fast_int_ok(num_layers, 1);
    for (int li = 0; li < num_layers; li++)
    {
        const tb200_layer_desc& L = layers[li];
        if (L.op != TB200_OP_CONV && L.op != TB200_OP_FC) continue;
        const TensorInfo& tin = g->tensors[L.inputs[0]];
        const TensorInfo& tout = g->tensors[L.output];
        const bool u8b = tin.d.data_type == TB200_DT_UINT8;
        const int OC = tout.d.dims[1];
        const size_t kk = L.op == TB200_OP_FC ? (size_t)tin.d.dims[1] * tin.d.dims[2] * tin.d.dims[3]
                                              : (size_t)(tin.d.dims[1] / L.group) * L.kernel_h * L.kernel_w;
        const int8_t* wsrc = (const int8_t*)L.weight;
        for (int o = 0; o < OC; o++)
        {
            double sumabs = 0;
            if (u8b)
                for (size_t k = 0; k < kk; k++) sumabs += abs((int)((const uint8_t*)L.weight)[(size_t)o * kk + k] - L.weight_zero);
            else
                for (size_t k = 0; k < kk; k++) sumabs += abs((int)wsrc[(size_t)o * kk + k]);
            const double M = (double)tin.d.scale * (double)L.weight_scales[u8b ? 0 : o] / (double)tout.d.scale;
            const double bound = ((u8b ? 255.0 : 128.0) * sumabs + fabs((double)(L.bias ? L.bias[o] : 0))) * fabs(M) + 256.0;
            if (!(bound < 32000.0)) fast_int_ok[li] = 0;
        }
    }

    // ---- pack weights into a host image of the arena, one H2D copy.  With a pack cache directory (tb200_pack_cache_dir /
    //      TG_B200_PACK_CACHE; SURVEY.md 8(f)-3) the image is keyed by a hash of everything it depends on -- descriptors, kernel
    //      choices, weights, biases, scales -- and a second prerun of the same model reads it back instead of packing again
    //      (the analogue of keeping conv_hcl_prerun's interleaved weights, conv_kernel_x86.c:2137-2209, next to the tmfile). ----
    if (!(flags & TB200_PRERUN_NO_WEIGHTS))
    {
        std::vector<uint8_t> img(g->w_bytes, 0);
        std::string cache_path;
        bool cache_hit = false;
        uint64_t cache_hash = 0;
        {
            const std::string dir = pack_cache_dir();
            if (!dir.empty())
            {
                uint64_t h = 1469598103934665603ull;
                auto mix = [&](const void* p, size_t n)
                {
                    const uint8_t* b = (const uint8_t*)p;
                    for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
                };
                const int ver = TB200_PACK_FORMAT * 16 + gemm_sx_mode();
                mix(&ver, sizeof ver), mix(&g->w_bytes, sizeof g->w_bytes), mix(&num_layers, sizeof num_layers);
                for (int li = 0; li < num_layers; li++)
                {
                    const tb200_layer_desc& L = layers[li];
                    mix(&kind[li], sizeof(int)), mix(&blobs[li], sizeof(WeightBlob)), mix(&fuse_bias[li], sizeof(int));
                    mix(&L.op, offsetof(tb200_layer_desc, weight)); // every scalar field up to the pointers
                    mix(&L.weight_zero, sizeof L.weight_zero), mix(&L.bias_scale, sizeof L.bias_scale);
                    for (int k = 0; k < L.num_inputs && k < 4; k++) mix(&g->tensors[L.inputs[k]].d, sizeof(tb200_tensor_desc));
                    if (L.op != TB200_OP_NOP_) mix(&g->tensors[L.output].d, sizeof(tb200_tensor_desc));
                    if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
                    {
                        const TensorInfo& ti = g->tensors[L.inputs[0]];
                        const TensorInfo& to = g->tensors[L.output];
                        const size_t kk = L.op == TB200_OP_FC ? (size_t)ti.d.dims[1] * ti.d.dims[2] * ti.d.dims[3]
                                                              : (size_t)(ti.d.dims[1] / L.group) * L.kernel_h * L.kernel_w;
                        mix(L.weight, (size_t)to.d.dims[1] * kk);
                        if (L.bias) mix(L.bias, (size_t)to.d.dims[1] * 4);
                        mix(L.weight_scales, ti.d.data_type == TB200_DT_UINT8 ? 4 : (size_t)to.d.dims[1] * 4);
                    }
                }
                // batch-dependent fields of the tensor descriptors were hashed too: a cache entry is per (model, batch) like a plan
                char name[64];
                snprintf(name, sizeof name, "/tb200_%016llx.pack", (unsigned long long)h);
                cache_path = dir + name;
                cache_hash = h;
                if (FILE* f = fopen(cache_path.c_str(), "rb"))
                {
                    uint64_t hdr[3] = {0, 0, 0};
                    if (fread(hdr, sizeof hdr, 1, f) == 1 && hdr[0] == 0x3032424b43415054ull + TB200_PACK_FORMAT && hdr[1] == h && hdr[2] == g->w_bytes &&
                        fread(img.data(), 1, g->w_bytes, f) == g->w_bytes)
                        cache_hit = true;
                    fclose(f);
                }
            }
        }
        g->pack_cache_state = cache_path.empty() ? 0 : (cache_hit ? 2 : 1);
        for (int li = 0; li < num_layers && !cache_hit; li++)
        {
            const tb200_layer_desc& L = layers[li];
            if (kind[li] == K_CONCAT_PART)
            {
                // per-input requantisation of concat_kernel_ref_int8.c:70-80 (roundf(q * (s_in / s_out)), including its clamp of
                // values below -127 to +127) and concat_kernel_ref_uint8.c:82 (roundf((q - zp_in) * (s_in / s_out) + zp_out), the zero
                // point inside the rounding, clamp) as byte tables
                const tb200_tensor_desc& to = g->tensors[L.output].d;
                for (int k = 0; k < L.num_inputs && k < 4; k++)
                {
                    const tb200_tensor_desc& ti = g->tensors[L.inputs[k]].d;
                    uint8_t* lut = img.data() + blobs[li].w_off + 256 * k;
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
                continue;
            }
            if (kind[li] == K_POOL && pool_relu[li] >= 0)
            {
                // tin = what the folded ReLU read, its own output quantisation = the pooling's
                build_relu_lut(g->tensors[L.inputs[0]].d.data_type == TB200_DT_UINT8, g->tensors[L.inputs[0]].d, g->tensors[L.output].d,
                               layers[pool_relu[li]].negative_slope, img.data() + blobs[li].w_off);
                continue;
            }
            if (kind[li] == K_LUT && L.op == TB200_OP_LUT2_)
            {
                // x -> sigmoid(x) (its own requantisation, the Sigmoid node's output tensor) -> eltwise product with x
                const tb200_layer_desc& S = src_layers[silu_sig[li]];
                const tb200_layer_desc& E = src_layers[li];
                const tb200_tensor_desc &tx = tensors[S.inputs[0]], &ts = tensors[S.output], &to = tensors[E.output];
                const bool u8l = tx.data_type == TB200_DT_UINT8;
                uint8_t sig[256];
                build_byte_lut(TB200_OP_SIGMOID, u8l, tx, ts, sig);
                uint8_t* lut = img.data() + blobs[li].w_off;
                for (int b = 0; b < 256; b++)
                    lut[b] = (E.inputs[0] == S.output) ? eltwise_byte(u8l, TB200_ELT_PROD, sig[b], ts, b, tx, to) : eltwise_byte(u8l, TB200_ELT_PROD, b, tx, sig[b], ts, to);
                continue;
            }
            if (kind[li] == K_LUT)
            {
                build_byte_lut(L.op, g->tensors[L.inputs[0]].d.data_type == TB200_DT_UINT8, g->tensors[L.inputs[0]].d, g->tensors[L.output].d,
                               img.data() + blobs[li].w_off);
                continue;
            }
            if (L.op != TB200_OP_CONV && L.op != TB200_OP_FC) continue;
            const TensorInfo& tin = g->tensors[L.inputs[0]];
            const TensorInfo& tout = g->tensors[L.output];
            const bool u8 = tin.d.data_type == TB200_DT_UINT8;
            const int C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3], OC = tout.d.dims[1];
            const uint8_t* src = (const uint8_t*)L.weight;
            uint8_t* dst = img.data() + blobs[li].w_off;
            const bool tc = kind[li] == K_GEMM || kind[li] == K_IGEMM;
            // row of output channel o in the packed B operand (uint8 tensor-core tiles carry 16 extra rows each)
            const int bn = tc ? gemm_block_n(tout.cp, u8) : tout.cp, bnx = tc ? gemm_tile_rows(tout.cp, u8 ? 1 + L.weight_zero : 0) : bn;
            auto brow = [&](int o) -> size_t { return (size_t)(o / bn) * bnx + (o % bn); };
            size_t krow = 0; // K extent of one packed row
            if (L.op == TB200_OP_FC)
            {
                // [OC][C*H*W] (NCHW flatten, fc_ref.c:313-359) -> [row][H][W][Cp]
                krow = (size_t)H * W * tin.cp;
                for (int o = 0; o < OC; o++)
                    for (int c = 0; c < C; c++)
                        for (int p = 0; p < H * W; p++) dst[(brow(o) * H * W + p) * tin.cp + c] = src[((size_t)o * C + c) * H * W + p];
            }
            else
            {
                const int KH = L.kernel_h, KW = L.kernel_w, cg = C / L.group;
                if (kind[li] == K_CONV_DW)
                {
                    for (int c = 0; c < C; c++)
                        for (int t = 0; t < KH * KW; t++) dst[(size_t)t * tin.cp + c] = src[(size_t)c * KH * KW + t];
                }
                else if (kind[li] == K_GATHER_TC && !(tin.input_index >= 0 && C <= 3))
                {
                    // 16- / 32-channel NHWC input: k = (kh*3 + kw)*Cp + c; rows of 160 bytes (the last 16 stay 0) / 288 bytes
                    const size_t rowb = tin.cp == 16 ? 160 : 288;
                    for (int o = 0; o < OC; o++)
                        for (int c = 0; c < C; c++)
                            for (int t = 0; t < 9; t++) dst[(size_t)o * rowb + t * tin.cp + c] = src[((size_t)o * C + c) * 9 + t];
                }
                else if (kind[li] == K_STEM_TC || kind[li] == K_GATHER_TC)
                {
                    // [OC][C][KH][KW] is already k = (c*KH + kh)*KW + kw order: one zero-padded row of 32*ks bytes per channel
                    const size_t kk = (size_t)C * KH * KW, kp = ((kk + 31) / 32) * 32;
                    for (int o = 0; o < OC; o++) memcpy(dst + (size_t)o * kp, src + (size_t)o * kk, kk);
                }
                else
                {
                    const int cgp = kind[li] == K_CONV_STEM ? 4 : (L.group == 1 ? tin.cp : cg);
                    krow = (size_t)KH * KW * cgp;
                    for (int o = 0; o < OC; o++)
                        for (int c = 0; c < cg; c++)
                            for (int t = 0; t < KH * KW; t++)
                                dst[(brow(o) * KH * KW + t) * cgp + c] = src[((size_t)o * cg + c) * KH * KW + t];
                }
            }
            std::vector<int64_t> wsum_tot(tout.cp, 0); // uint8 tensor-core kinds: sum of the raw weight bytes per channel
            if (tc && u8)
            {
                // the tensor cores form sum x*(w - zw) themselves: B = w - 128 as int8 (plus a constant tile of 128 - zw in the kernel),
                // or plain w when zw == 0.  Real K positions only; pad positions stay 0 (x is 0 there anyway).
                if (L.weight_zero != 0)
                {
                    const size_t kreal_row = krow; // bytes per packed row
                    for (int o = 0; o < OC; o++)
                    {
                        uint8_t* row = dst + brow(o) * kreal_row;
                        if (L.op == TB200_OP_FC)
                        {
                            for (int c = 0; c < C; c++)
                                for (int p2 = 0; p2 < H * W; p2++) row[(size_t)p2 * tin.cp + c] = (uint8_t)(int8_t)((int)row[(size_t)p2 * tin.cp + c] - 128);
                        }
                        else
                        {
                            const int KT = L.kernel_h * L.kernel_w;
                            for (int t = 0; t < KT; t++)
                                for (int c = 0; c < C; c++) row[(size_t)t * tin.cp + c] = (uint8_t)(int8_t)((int)row[(size_t)t * tin.cp + c] - 128);
                        }
                    }
                }
                if (bnx != bn) // sum(x) of every pixel from the main MMA: 16 rows of ones close every B tile (gemm_tcgen05.cu, sx_mode 0)
                    for (int tile = 0; tile * bn < tout.cp; tile++) memset(dst + ((size_t)tile * bnx + bn) * krow, 1, (size_t)16 * krow);
                const int taps = L.op == TB200_OP_FC ? 1 : L.kernel_h * L.kernel_w;
                const int kk = L.op == TB200_OP_FC ? C * H * W : C; // real K elements per tap
                std::vector<int64_t> tapc((size_t)taps * OC, 0); // what a tap that falls into the padding must give back: zx*(sum_c w - Cin*zw)
                for (int o = 0; o < OC; o++)
                    for (int t = 0; t < taps; t++)
                    {
                        int64_t sw = 0;
                        if (L.op == TB200_OP_FC)
                            for (int k = 0; k < kk; k++) sw += src[(size_t)o * kk + k];
                        else
                            for (int c = 0; c < C; c++) sw += src[((size_t)o * C + c) * taps + t];
                        wsum_tot[o] += sw;
                        tapc[(size_t)t * OC + o] = (int64_t)tin.d.zero_point * (sw - (int64_t)kk * L.weight_zero);
                    }
                if (kind[li] == K_IGEMM)
                {
                    // Border patterns: a pixel whose window is cut by a rows at the top, b at the bottom, c columns on the left and d on
                    // the right misses the taps {kh < a or kh >= KH-b or kw < c or kw >= KW-d}; the table holds the SUM of their
                    // corrections per channel, index ((a*(KH+1) + b)*(pw+1) + c)*(KW+1) + d (gemm_tcgen05.cu border_pattern), so a
                    // border row costs one vector load per four channels instead of a loop over taps.
                    const int KH = L.kernel_h, KW = L.kernel_w;
                    int32_t* pt = (int32_t*)(img.data() + blobs[li].btab_off);
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
            }
            if (kind[li] == K_GATHER_TC && u8)
            {
                const int kk = C * L.kernel_h * L.kernel_w;
                for (int o = 0; o < OC; o++)
                    for (int k = 0; k < kk; k++) wsum_tot[o] += src[(size_t)o * kk + k];
            }
            int32_t* b = (int32_t*)(img.data() + blobs[li].bias_off);
            float* sc = (float*)(img.data() + blobs[li].scale_off);
            float* fm = (float*)(img.data() + blobs[li].fast_off); // float2 per channel: (multiplier | bias term, bias bits)
            const bool fc = L.op == TB200_OP_FC;
            const bool fuse = fuse_bias[li] != 0;
            for (int o = 0; o < tout.cp; o++)
            {
                b[o] = (L.bias && o < OC) ? L.bias[o] : 0;
                sc[o] = u8 ? L.weight_scales[0] : (o < OC ? L.weight_scales[o] : 1.f);
                if (u8 && (tc || kind[li] == K_GATHER_TC))
                {
                    // tensor-core layers: the int8 layout { M[2k], M[2k+1], y[2k], y[2k+1] } with y = corr[oc] + bias[oc] as an integer
                    // (corr[oc] = -zx*sum_k w + K*zx*zw: what the zero points contribute when every tap is inside the image)
                    float* fmM = fm + (size_t)(o >> 1) * 4 + (o & 1);
                    float* fmY = fmM + 2;
                    int32_t y = 0;
                    if (o < OC)
                    {
                        const int64_t kreal = fc ? (int64_t)C * H * W : (int64_t)C * L.kernel_h * L.kernel_w;
                        y = (int32_t)(-(int64_t)tin.d.zero_point * wsum_tot[o] + kreal * tin.d.zero_point * L.weight_zero + (int64_t)b[o]);
                    }
                    *fmM = (o >= OC) ? 0.f : (float)((double)tin.d.scale * (double)L.weight_scales[0] / (double)tout.d.scale);
                    memcpy(fmY, &y, 4);
                }
                else if (u8)
                {
                    // the bias term in real units, rounded exactly as the reference rounds it
                    const float S = tin.d.scale * L.weight_scales[0];
                    // FC: fc_ref.c:141-146 multiplies by the BIAS TENSOR's own scale (normally s_in*s_w, but the file decides)
                    const float Sb = (fc && L.bias_scale != 0.f) ? L.bias_scale : S;
                    fm[2 * o] = (o >= OC) ? 0.f : (fc ? (float)b[o] * Sb : ((L.recipe == TB200_RECIPE_HCL) ? (float)b[o] * S : ((float)b[o] * tin.d.scale) * L.weight_scales[0]));
                    // tensor-core kinds: corr[oc] = -zx*sum_k w + K*zx*zw (all taps in bounds), carried in the .y lane
                    int32_t corr = 0;
                    if ((tc || kind[li] == K_GATHER_TC) && o < OC)
                    {
                        const int64_t kreal = fc ? (int64_t)C * H * W : (int64_t)C * L.kernel_h * L.kernel_w;
                        corr = (int32_t)(-(int64_t)tin.d.zero_point * wsum_tot[o] + kreal * tin.d.zero_point * L.weight_zero);
                    }
                    memcpy(&fm[2 * o + 1], &corr, 4);
                }
                else
                {
                    // channel pairs interleaved (common.cuh FastPar4): { M[2k], M[2k+1], y[2k], y[2k+1] }
                    float* fmM = fm + (size_t)(o >> 1) * 4 + (o & 1);
                    float* fmY = fmM + 2;
                    if (o >= OC) *fmM = 0.f;
                    else if (fc) *fmM = (tin.d.scale * sc[o]) / tout.d.scale; // fc_ref.c:225, the reference's own requant scale
                    else *fmM = (float)((double)tin.d.scale * (double)sc[o] / (double)tout.d.scale);
                    if (fuse) *fmY = (o >= OC) ? 0.f : (float)((double)b[o] * (double)*fmM); // fl(bias*M)
                    else memcpy(fmY, &b[o], 4);
                }
            }
        }
        if (getenv("TB200_DEBUG_HASH") && atoi(getenv("TB200_DEBUG_HASH")) >= 2)
        {
            auto fnv = [](const void* p, size_t n) {
                uint64_t h = 1469598103934665603ull;
                for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
                return (unsigned long long)h;
            };
            for (int li = 0; li < num_layers; li++)
            {
                const tb200_layer_desc& L = layers[li];
                if (L.op != TB200_OP_CONV && L.op != TB200_OP_FC) continue;
                const int ocp = g->tensors[L.output].cp;
                {
                    const float* fmv = (const float*)(img.data() + blobs[li].fast_off);
                    const TensorInfo& ti = g->tensors[L.inputs[0]];
                    const TensorInfo& to = g->tensors[L.output];
                    int y0, y1;
                    memcpy(&y0, fmv + 2, 4), memcpy(&y1, fmv + 3, 4);
                    fprintf(stderr, "[tb200 dbg] pack layer %d consts: in(%.9g, %d) out(%.9g, %d) ws %.9g wz %d M %.9g %.9g y %d %d bias0 %d\n", li, ti.d.scale, ti.d.zero_point,
                            to.d.scale, to.d.zero_point, L.weight_scales[0], L.weight_zero, fmv[0], fmv[1], y0, y1, L.bias ? L.bias[0] : 0);
                }
                fprintf(stderr, "[tb200 dbg] pack layer %d kind %d: w %016llx (%zu) bias %016llx scale %016llx fast %016llx fuse %d fast_int %d u8fast %d\n", li, kind[li],
                        fnv(img.data() + blobs[li].w_off, blobs[li].w_size), blobs[li].w_size, fnv(img.data() + blobs[li].bias_off, (size_t)ocp * 4),
                        fnv(img.data() + blobs[li].scale_off, (size_t)ocp * 4), fnv(img.data() + blobs[li].fast_off, (size_t)ocp * 8), fuse_bias[li], fast_int_ok[li],
                        u8_tc_fast[li]);
            }
        }
        if (!cache_path.empty() && !cache_hit)
        {
            // write-then-rename so that a concurrent reader never sees a partial file; failure to write is not an error
            const std::string tmp = cache_path + ".tmp" + std::to_string((long long)getpid());
            if (FILE* f = fopen(tmp.c_str(), "wb"))
            {
                const uint64_t hdr[3] = {0x3032424b43415054ull + TB200_PACK_FORMAT, cache_hash, g->w_bytes};
                const bool ok = fwrite(hdr, sizeof hdr, 1, f) == 1 && fwrite(img.data(), 1, g->w_bytes, f) == g->w_bytes;
                fclose(f);
                if (!ok || rename(tmp.c_str(), cache_path.c_str()) != 0) remove(tmp.c_str());
            }
        }
        CUDA_OK(cudaMemcpyAsync(g->w_arena, img.data(), g->w_bytes, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_OK(cudaStreamSynchronize(ctx->stream));
    }

    // ---- build the launch sequence: the batch is cut into K equal chunks (images are independent units) so that `run`
    //      can overlap the H2D copy of chunk i+1 with the kernels of chunk i; each chunk owns a slice of every tensor ----
    int Ntot = g->tensors[0].d.dims[0];
    bool same_batch = true;
    for (auto& t : g->tensors) same_batch &= (t.d.dims[0] == Ntot);
    int K = 1;
    std::vector<int> cfirst{0}, ccount{Ntot};
    if (same_batch && !(flags & TB200_PRERUN_NO_GRAPH))
    {
        K = Ntot >= 32 ? 2 : 1;
        if (const char* ev = getenv("TB200_PIPELINE_CHUNKS")) K = atoi(ev) > 0 ? atoi(ev) : K;
        while (K > 1 && Ntot % K) K--;
        cfirst.clear(), ccount.clear();
        for (int k = 0; k < K; k++) cfirst.push_back(k * (Ntot / K)), ccount.push_back(Ntot / K);
        if (K == 2 && Ntot >= 64 && !getenv("TB200_PIPELINE_CHUNKS"))
        {
            // two chunks of 1/4 and 3/4: the kernels only ever wait for the first quarter of the input (measured on MobileNet-v1
            // b=256 through tb200_graph_run: 1.78 ms vs 1.92 ms for two halves; three-way splits 1.85-1.87 ms)
            const int a = ((Ntot / 4 + 7) / 8) * 8;
            cfirst = {0, a}, ccount = {a, Ntot - a};
        }
        // TB200_PIPELINE_SPLIT="40,88,128": explicit (uneven) chunk sizes in images -- a small first chunk shortens the time the
        // kernels wait for the first H2D copy; must sum to the batch
        if (const char* ev = getenv("TB200_PIPELINE_SPLIT"))
        {
            std::vector<int> sz;
            int sum = 0;
            for (const char* p = ev; *p;)
            {
                char* end;
                const long v = strtol(p, &end, 10);
                if (end == p || v <= 0) break;
                sz.push_back((int)v), sum += (int)v;
                p = (*end == ',') ? end + 1 : end;
            }
            if (sum == Ntot && sz.size() >= 1 && sz.size() <= 16)
            {
                cfirst.clear(), ccount.clear(), K = (int)sz.size();
                int f = 0;
                for (int v : sz) cfirst.push_back(f), ccount.push_back(v), f += v;
            }
        }
    }
    const int Kpipe = K;
    g->chunks = Kpipe;
    g->chunk_first = cfirst, g->chunk_count = ccount;
    g->chunk_steps.resize(Kpipe > 1 ? Kpipe : 0);
    // builds the launch sequence of images [first, first + nb) (the whole batch, or one pipeline chunk) into `steps`
    auto build_steps = [&](const int first, const int nb, std::vector<Step>& steps, const bool count_work) -> int
    {
        // byte offset of image `first` inside a tensor of the whole batch
        auto img_off = [&](size_t total_bytes) -> size_t { return (total_bytes / (size_t)Ntot) * (size_t)first; };
        auto tdev = [&](const TensorInfo& t) -> uint8_t* { return t.dev + img_off(t.nhwc_bytes); };
        for (size_t i = 0; i < g->input_ids.size(); i++)
        {
            TensorInfo& t = g->tensors[g->input_ids[i]];
            if (!t.nhwc_needed) continue;
            Step s;
            s.kind = K_NCHW2NHWC, s.layer = -1, s.in = g->in_nchw_dev[i] + img_off(t.nchw_bytes), s.out = tdev(t);
            s.n = nb, s.c = t.d.dims[1], s.h = t.d.dims[2], s.w_ = t.d.dims[3];
            steps.push_back(s);
        }
        for (int li = 0; li < num_layers; li++)
        {
            const tb200_layer_desc& L = layers[li];
            if (L.op == TB200_OP_NOP_)
            {
                g->layer_kernel[li] = kStepName[K_NONE];
                continue;
            }
            TensorInfo& tin = g->tensors[L.inputs[0]];
            TensorInfo& tout = g->tensors[L.output];
            const bool u8 = tin.d.data_type == TB200_DT_UINT8;
            Step s;
            s.kind = kind[li], s.layer = li, s.u8 = u8;
            s.in = tdev(tin), s.out = tdev(tout);
            const int N = nb, C = tin.d.dims[1], H = tin.d.dims[2], W = tin.d.dims[3];
            const int OC = tout.d.dims[1], OH = tout.d.dims[2], OW = tout.d.dims[3];
            if (L.op == TB200_OP_CONV || L.op == TB200_OP_FC)
            {
                const bool fc = L.op == TB200_OP_FC;
                s.w = g->w_arena + blobs[li].w_off;
                s.epi = make_epi(L, tin.d, tout.d, fc);
                s.epi.bias = (const int32_t*)(g->w_arena + blobs[li].bias_off);
                s.epi.w_scale = (const float*)(g->w_arena + blobs[li].scale_off);
                s.epi.fast_par = (const float2*)(g->w_arena + blobs[li].fast_off);
                s.btab = (const int32_t*)(g->w_arena + blobs[li].btab_off);
                s.epi.fuse_bias = fuse_bias[li];
                if (!fast_int_ok[li] || !u8_tc_fast[li]) s.epi.fast_ok = 0;
                ConvShape& cs = s.cs;
                cs.n = N, cs.h = H, cs.w = W, cs.c = C, cs.cp = tin.cp, cs.oh = OH, cs.ow = OW, cs.oc = OC, cs.ocp = tout.cp;
                if (fc)
                {
                    cs.kh = H, cs.kw = W, cs.sh = cs.sw = 1, cs.ph0 = cs.pw0 = 0, cs.dh = cs.dw = 1, cs.group = 1;
                    cs.cg = C, cs.cgp = tin.cp;
                    if (count_work)
                    {
                        g->work_ops += 2.0 * Ntot * OC * C * H * W;
                        g->work_bytes += (double)tin.nchw_bytes + tout.nchw_bytes + (double)OC * C * H * W + (L.bias ? 4.0 * OC : 0);
                        g->work_wbytes += (double)OC * C * H * W + (L.bias ? 4.0 * OC : 0);
                    }
                }
                else
                {
                    cs.kh = L.kernel_h, cs.kw = L.kernel_w, cs.sh = L.stride_h, cs.sw = L.stride_w, cs.ph0 = L.pad_h0, cs.pw0 = L.pad_w0;
                    cs.dh = L.dilation_h, cs.dw = L.dilation_w, cs.group = L.group;
                    cs.cg = C / L.group, cs.cgp = (L.group == 1) ? tin.cp : cs.cg;
                    const double k = (double)cs.cg * cs.kh * cs.kw;
                    if (count_work)
                    {
                        g->work_ops += 2.0 * (double)tout.nchw_bytes * k;
                        g->work_bytes += (double)tin.nchw_bytes + tout.nchw_bytes + (double)OC * k + (L.bias ? 4.0 * OC : 0);
                        g->work_wbytes += (double)OC * k + (L.bias ? 4.0 * OC : 0);
                    }
                }
                if (s.kind == K_CONV_STEM || s.kind == K_STEM_TC || (s.kind == K_GATHER_TC && tin.input_index >= 0 && C <= 3))
                    s.in = g->in_nchw_dev[tin.input_index] + img_off(tin.nchw_bytes);
                s.nhwc16 = (s.kind == K_GATHER_TC && !(tin.input_index >= 0 && C <= 3)) ? 1 : 0;
                if (s.kind == K_STEM_TC) stem_plan_create(&s.dwp, s.in, s.cs); // falls back to the global-memory gather
                if (s.kind == K_GATHER_TC)
                {
                    window_plan_create(&s.wp, s.in, s.cs, s.nhwc16); // falls back to the global-memory gather (16 channels / NCHW only)
                    if (!s.wp.valid && s.nhwc16 && tin.cp != 16) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: window plan failed for a 32-channel 3x3 convolution", li));
                }
                if (s.kind == K_CONV_DW && !(flags & TB200_PRERUN_NO_TENSORCORE)) dw_plan_create(&s.dwp, s.in, s.cs, s.epi); // falls back when not applicable
                if (s.kind == K_IGEMM)
                {
                    int rc = gemm_plan_create_conv(&s.gemm, s.in, s.w, s.out, s.cs, u8 ? 1 + L.weight_zero : 0);
                    if (rc) return bail(fail(rc, "layer %d: implicit-GEMM plan failed", li));
                    s.gemm.fixq = ctx->fixq, s.gemm.fixq_cap = FIXQ_CAP;
                }
                if (s.kind == K_GEMM)
                {
                    const long long m = fc ? N : (long long)N * H * W;
                    const int kdim = fc ? H * W * tin.cp : tin.cp;
                    int rc = gemm_plan_create(&s.gemm, s.in, kdim, s.w, s.out, m, kdim, OC, tout.cp, tout.cp, 0, u8 ? 1 + L.weight_zero : 0);
                    if (rc) return bail(fail(rc, "layer %d: TMA descriptor creation failed (m=%lld k=%d oc=%d)", li, m, kdim, OC));
                    s.gemm.fixq = ctx->fixq, s.gemm.fixq_cap = FIXQ_CAP;
                }
            }
            else if (L.op == TB200_OP_POOL)
            {
                PoolShape& p = s.ps;
                p.n = N, p.h = H, p.w = W, p.c = C, p.cp = tin.cp, p.oh = OH, p.ow = OW;
                p.kh = L.kernel_h, p.kw = L.kernel_w, p.sh = L.stride_h, p.sw = L.stride_w, p.ph0 = L.pad_h0, p.pw0 = L.pad_w0;
                p.method = L.pool_method, p.caffe_flavor = L.caffe_flavor;
                p.in_scale = tin.d.scale, p.out_scale = tout.d.scale, p.in_zero = tin.d.zero_point, p.out_zero = tout.d.zero_point;
                if (L.pool_global) p.kh = H, p.kw = W, p.sh = p.sw = 1, p.ph0 = p.pw0 = 0;
                p.lut = pool_relu[li] >= 0 ? g->w_arena + blobs[li].w_off : nullptr, p.c_real = u8 ? C : tin.cp;
                if (tout.d.dims[1] != C) return bail(fail(TB200_ERR_INVALID, "layer %d: pool channel mismatch", li));
            }
            else if (L.op == TB200_OP_RELU || L.op == TB200_OP_ELTWISE)
            {
                PointwiseParams& p = s.pp;
                p.c = C, p.cp = tin.cp;
                p.scale0 = tin.d.scale, p.zero0 = tin.d.zero_point, p.out_scale = tout.d.scale, p.out_zero = tout.d.zero_point;
                p.negative_slope = L.negative_slope;
                p.post_relu = post_relu[li], p.post_floor4 = (uint32_t)(tout.d.zero_point & 0xff) * 0x01010101u;
                if (L.op == TB200_OP_RELU)
                    p.mode = 0, p.scale1 = 0, p.zero1 = 0;
                else
                {
                    const TensorInfo& t1 = g->tensors[L.inputs[1]];
                    if (t1.nhwc_bytes != tin.nhwc_bytes) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: eltwise broadcast", li));
                    p.mode = L.elt_type == TB200_ELT_SUM ? 1 : 2;
                    p.scale1 = t1.d.scale, p.zero1 = t1.d.zero_point;
                    s.in2 = tdev(t1);
                }
                s.bytes = (long long)(tin.nhwc_bytes / (size_t)Ntot * (size_t)nb);
                if (tout.nhwc_bytes != tin.nhwc_bytes) return bail(fail(TB200_ERR_INVALID, "layer %d: pointwise shape mismatch", li));
            }
            else if (L.op == TB200_OP_CONCAT && L.num_inputs > 1)
            {
                int coff = 0;
                for (int k = 0; k < L.num_inputs; k++)
                {
                    const TensorInfo& tk = g->tensors[L.inputs[k]];
                    Step p = s;
                    p.in = tdev(tk);
                    p.npix = (long long)N * H * W, p.c = tk.d.dims[1], p.cp_in = tk.cp, p.cp_out = tout.cp, p.c_off = coff;
                    p.s_in = tk.d.scale, p.z_in = tk.d.zero_point, p.s_out = tout.d.scale, p.z_out = tout.d.zero_point;
                    p.c_write = (k + 1 == L.num_inputs) ? tout.cp - coff : tk.d.dims[1];
                    // vectorised table path when everything is 16-channel aligned; identical quantisation -> no table at all
                    p.scale = (tk.d.dims[1] % 16 == 0 && coff % 16 == 0 && !getenv("TB200_CONCAT_BYTEWISE")) ? 1 : 0;
                    p.w = (tk.d.scale == tout.d.scale && tk.d.zero_point == tout.d.zero_point) ? nullptr : g->w_arena + blobs[li].w_off + 256 * k;
                    coff += tk.d.dims[1];
                    if (k + 1 < L.num_inputs) steps.push_back(p);
                    else s = p;
                }
                if (coff != OC) return bail(fail(TB200_ERR_INVALID, "layer %d: concat channels %d != %d", li, coff, OC));
            }
            else if (L.op == TB200_OP_UPSAMPLE)
            {
                s.n = N, s.h = H, s.w_ = W, s.cp_in = tin.cp, s.scale = L.up_scale;
                if (OH != H * L.up_scale || OW != W * L.up_scale) return bail(fail(TB200_ERR_INVALID, "layer %d: upsample shape", li));
            }
            else if (s.kind == K_LUT)
            {
                s.w = g->w_arena + blobs[li].w_off;
                s.bytes = (long long)(tin.nhwc_bytes / (size_t)Ntot * (size_t)nb);
                s.c = C, s.cp_in = tin.cp;
                if (tout.nhwc_bytes != tin.nhwc_bytes) return bail(fail(TB200_ERR_INVALID, "layer %d: unary op changes the shape", li));
            }
            else if (s.kind == K_SOFTMAX)
            {
                if (tout.nhwc_bytes != tin.nhwc_bytes) return bail(fail(TB200_ERR_INVALID, "layer %d: softmax changes the shape", li));
                s.npix = (long long)N * H * W, s.c = C, s.cp_in = tin.cp;
                s.s_in = tin.d.scale, s.z_in = tin.d.zero_point, s.s_out = tout.d.scale, s.z_out = tout.d.zero_point;
            }
            else if (s.kind == K_RESHAPE)
            {
                s.n = N, s.c = C, s.h = H, s.w_ = W, s.oc_ = OC, s.oh_ = OH, s.ow_ = OW;
                s.scratch = g->act_arena + scratch_off[li]; // NCHW-ordered bytes of this chunk (chunks never run concurrently)
            }
            else if (L.op == TB200_OP_IDENTITY || L.op == TB200_OP_CONCAT || L.op == TB200_OP_RESHAPE)
            {
                s.bytes = (long long)(tin.nhwc_bytes / (size_t)Ntot * (size_t)nb);
                if (tout.nhwc_bytes != tin.nhwc_bytes) return bail(fail(TB200_ERR_UNSUPPORTED, "layer %d: identity changes the NHWC footprint", li));
            }
            g->layer_kernel[li] = (s.kind == K_CONV_DW && s.dwp.valid) ? "conv_dw3x3_tma_dp4a" : ((s.kind == K_GATHER_TC && s.wp.valid) ? "conv_window_tcgen05" : kStepName[s.kind]);
            steps.push_back(s);
        }
        for (size_t i = 0; i < g->output_ids.size(); i++)
        {
            TensorInfo& t = g->tensors[g->output_ids[i]];
            Step s;
            s.kind = K_NHWC2NCHW, s.layer = -1, s.in = tdev(t), s.out = g->out_nchw_dev[i] + img_off(t.nchw_bytes);
            s.n = nb, s.c = t.d.dims[1], s.h = t.d.dims[2], s.w_ = t.d.dims[3];
            steps.push_back(s);
        }
        return 0;
    };
    // the whole-batch plan serves tb200_graph_launch / profile (device-resident use); the chunk plans serve the pipelined
    // tb200_graph_run.  They address the same tensors (a chunk is a slice of dim 0), so either may run at any time.
    {
        int rc = build_steps(0, Ntot, g->steps, true);
        if (rc) return rc;
        for (int ck = 0; ck < (int)g->chunk_steps.size(); ck++)
            if ((rc = build_steps(cfirst[ck], ccount[ck], g->chunk_steps[ck], false)) != 0) return rc;
    }
    g->num_launches = (int)g->steps.size();
    for (const Step& st : g->steps) g->num_launches += st.kind == K_RESHAPE ? 1 : 0; // two layout kernels
    CUDA_OK(cudaStreamSynchronize(ctx->stream));

    // ---- capture the launch sequences into CUDA graphs: [0] = whole batch, [1..K] = the pipeline chunks ----
    if (!(flags & TB200_PRERUN_NO_GRAPH))
    {
        const int ngraphs = 1 + (int)g->chunk_steps.size();
        g->cu_graphs.assign(ngraphs, nullptr);
        g->cu_execs.assign(ngraphs, nullptr);
        for (int gi = 0; gi < ngraphs; gi++)
        {
            const std::vector<Step>& seq = gi == 0 ? g->steps : g->chunk_steps[gi - 1];
            CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
            int rc = 0;
            for (const Step& s : seq)
                if ((rc = run_step(g, s, ctx->stream)) != 0) break;
            cudaError_t ce = cudaStreamEndCapture(ctx->stream, &g->cu_graphs[gi]);
            if (rc) return bail(rc);
            if (ce != cudaSuccess) return bail(fail(TB200_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce)));
            ce = cudaGraphInstantiate(&g->cu_execs[gi], g->cu_graphs[gi], 0);
            if (ce != cudaSuccess) return bail(fail(TB200_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(ce)));
        }
        const int K = Kpipe;
        if (K > 1)
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
    }
    return 0;
}

// ---- page-locking of the caller's buffers ---------------------------------------------------------------------------------
// Tengine hands `run` the application's malloc'd NCHW buffers (ir_tensor->data, c_api.c:1141-1160).  A cudaMemcpyAsync from
// pageable memory is staged by the driver and blocks the calling thread, which would serialise the GPUs of a group and the
// chunks of the copy/compute pipeline.  So a buffer is registered (cudaHostRegisterPortable) the first time it is seen and the
// registration is cached (up to 16 ranges, oldest dropped; everything is unregistered at postrun / context destruction).
// Returns true when [p, p+bytes) is page-locked.  Failure is not an error: the copy then takes the driver's pageable path.
static bool host_pin(tb200_context* root, const void* ptr, size_t bytes)
{
    static const bool off = getenv("TB200_NO_HOST_REGISTER") != nullptr;
    if (off || !ptr || !bytes) return false;
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
static inline size_t image_bytes(const tb200_graph* g, int tensor_id) { return g->tensors[tensor_id].nchw_bytes / (size_t)g->num_images; }

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
        // a failed CUDA call may have left a capture open on the context stream
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(ctx->stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone)
        {
            cudaGraph_t junk = nullptr;
            cudaStreamEndCapture(ctx->stream, &junk);
            if (junk) cudaGraphDestroy(junk);
        }
        cudaGetLastError();
        destroy_graph(g);
        return rc;
    }
    g->num_images = g->total_images = tensors[0].dims[0];
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
        sh->first_image = first, sh->num_images = count, sh->total_images = N;
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
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const int id = sh->input_ids[input_index];
        CUDA_OK(cudaMemcpyAsync(sh->in_nchw_dev[input_index], (const uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, id),
                                sh->tensors[id].nchw_bytes, cudaMemcpyHostToDevice, sh->ctx->stream));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

static unsigned long long debug_fnv(const void* p, size_t n)
{
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
    return (unsigned long long)h;
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
        fprintf(stderr, "[tb200 dbg] weight arena %zu bytes hash %016llx\n", g->w_bytes, debug_fnv(host.data(), g->w_bytes));
        for (const Step& s : g->steps)
        {
            int rc = run_step(g, s, g->ctx->stream);
            if (rc) return rc;
            CUDA_OK(cudaStreamSynchronize(g->ctx->stream));
            if (s.layer < 0) continue;
            const TensorInfo& t = g->tensors[g->layers[s.layer].output];
            host.resize(t.nhwc_bytes);
            CUDA_OK(cudaMemcpy(host.data(), t.dev, t.nhwc_bytes, cudaMemcpyDeviceToHost));
            fprintf(stderr, "[tb200 dbg] layer %d %s out [%d %d %d %d] hash %016llx\n", s.layer, kStepName[s.kind], t.d.dims[0], t.d.dims[1], t.d.dims[2], t.d.dims[3],
                    debug_fnv(host.data(), t.nhwc_bytes));
        }
        return 0;
    }
    if (!g->cu_execs.empty())
    {
        CUDA_OK(cudaGraphLaunch(g->cu_execs[0], g->ctx->stream)); // the whole-batch graph
        return 0;
    }
    for (const Step& s : g->steps)
    {
        int rc = run_step(g, s, g->ctx->stream);
        if (rc) return rc;
    }
    return 0;
}

int tb200_graph_launch(tb200_graph* g)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) { return launch_one(sh); });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_download(tb200_graph* g, int output_index, void* host_nchw)
{
    if (!g || output_index < 0 || output_index >= (int)g->output_ids.size() || !host_nchw) return fail(TB200_ERR_INVALID, "bad download arguments");
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const int id = sh->output_ids[output_index];
        CUDA_OK(cudaMemcpyAsync((uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, id), sh->out_nchw_dev[output_index],
                                sh->tensors[id].nchw_bytes, cudaMemcpyDeviceToHost, sh->ctx->stream));
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
static int run_enqueue_h2d(tb200_graph* g, const void* const* host_inputs)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    if (g->chunks <= 1 || g->cu_execs.empty())
    {
        for (size_t i = 0; i < g->input_ids.size(); i++)
        {
            const int id = g->input_ids[i];
            CUDA_OK(cudaMemcpyAsync(g->in_nchw_dev[i], (const uint8_t*)host_inputs[i] + (size_t)g->first_image * image_bytes(g, id),
                                    g->tensors[id].nchw_bytes, cudaMemcpyHostToDevice, g->ctx->stream));
        }
        return 0;
    }
    // Pipelined: the H2D copies of all chunks are queued back to back on the copy stream (the link stays busy), chunk k's
    // kernels start as soon as ITS slice has landed, and its outputs leave on a third stream while chunk k+1 computes.
    const int K = g->chunks;
    CUDA_OK(cudaEventRecord(g->ev_done, g->ctx->stream)); // order after whatever the caller queued on the context stream
    CUDA_OK(cudaStreamWaitEvent(g->copy_stream, g->ev_done, 0));
    for (int ck = 0; ck < K; ck++)
    {
        for (size_t i = 0; i < g->input_ids.size(); i++)
        {
            const int id = g->input_ids[i];
            const size_t ib = image_bytes(g, id), off = ib * (size_t)g->chunk_first[ck], bytes = ib * (size_t)g->chunk_count[ck];
            CUDA_OK(cudaMemcpyAsync(g->in_nchw_dev[i] + off, (const uint8_t*)host_inputs[i] + (size_t)g->first_image * ib + off, bytes, cudaMemcpyHostToDevice,
                                    g->copy_stream));
        }
        CUDA_OK(cudaEventRecord(g->ev_in[ck], g->copy_stream));
    }
    return 0;
}
// (2) kernels + D2H
static int run_enqueue_compute(tb200_graph* g, void* const* host_outputs)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    cudaStream_t cs = g->ctx->stream;
    static const int dbg2 = getenv("TB200_DEBUG_HASH") ? atoi(getenv("TB200_DEBUG_HASH")) : 0;
    if (g->chunks <= 1 || g->cu_execs.empty() || dbg2 >= 2)
    {
        int rc = launch_one(g);
        if (rc) return rc;
        for (size_t i = 0; i < g->output_ids.size(); i++)
        {
            const int id = g->output_ids[i];
            CUDA_OK(cudaMemcpyAsync((uint8_t*)host_outputs[i] + (size_t)g->first_image * image_bytes(g, id), g->out_nchw_dev[i], g->tensors[id].nchw_bytes,
                                    cudaMemcpyDeviceToHost, cs));
        }
        return 0;
    }
    const int K = g->chunks;
    for (int ck = 0; ck < K; ck++)
    {
        CUDA_OK(cudaStreamWaitEvent(cs, g->ev_in[ck], 0));
        CUDA_OK(cudaGraphLaunch(g->cu_execs[1 + ck], cs));
        CUDA_OK(cudaEventRecord(g->ev_out[ck], cs));
        CUDA_OK(cudaStreamWaitEvent(g->d2h_stream, g->ev_out[ck], 0));
        for (size_t i = 0; i < g->output_ids.size(); i++)
        {
            const int id = g->output_ids[i];
            const size_t ib = image_bytes(g, id), off = ib * (size_t)g->chunk_first[ck], bytes = ib * (size_t)g->chunk_count[ck];
            CUDA_OK(cudaMemcpyAsync((uint8_t*)host_outputs[i] + (size_t)g->first_image * ib + off, g->out_nchw_dev[i] + off, bytes, cudaMemcpyDeviceToHost,
                                    g->d2h_stream));
        }
    }
    return 0;
}
// (3) wait
static int run_wait(tb200_graph* g)
{
    CUDA_OK(cudaSetDevice(g->ctx->device));
    if (g->d2h_stream && g->chunks > 1 && !g->cu_execs.empty()) CUDA_OK(cudaStreamSynchronize(g->d2h_stream));
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
    for (size_t i = 0; i < g->input_ids.size(); i++) host_pin(g->ctx, host_inputs[i], image_bytes(g, g->input_ids[i]) * (size_t)g->total_images);
    for (size_t i = 0; i < g->output_ids.size(); i++) host_pin(g->ctx, host_outputs[i], image_bytes(g, g->output_ids[i]) * (size_t)g->total_images);
    int rc = for_each_shard(g, [&](tb200_graph* sh, int) { return run_enqueue_h2d(sh, host_inputs); });
    if (!rc) rc = for_each_shard(g, [&](tb200_graph* sh, int) { return run_enqueue_compute(sh, host_outputs); });
    const int rc2 = for_each_shard(g, [&](tb200_graph* sh, int) { return run_wait(sh); }); // always drain what was queued
    cudaSetDevice(g->ctx->device);
    static const bool dbg = getenv("TB200_DEBUG_HASH") != nullptr;
    if (dbg)
    {
        auto fnv = [](const void* p, size_t n) {
            uint64_t h = 1469598103934665603ull;
            for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
            return (unsigned long long)h;
        };
        for (size_t i = 0; i < g->input_ids.size(); i++)
            fprintf(stderr, "[tb200 run] input %zu: %zu bytes, hash %016llx\n", i, image_bytes(g, g->input_ids[i]) * (size_t)g->total_images,
                    fnv(host_inputs[i], image_bytes(g, g->input_ids[i]) * (size_t)g->total_images));
        for (size_t i = 0; i < g->output_ids.size(); i++)
            fprintf(stderr, "[tb200 run] output %zu (tensor %d): %zu bytes, hash %016llx\n", i, g->output_ids[i], image_bytes(g, g->output_ids[i]) * (size_t)g->total_images,
                    fnv(host_outputs[i], image_bytes(g, g->output_ids[i]) * (size_t)g->total_images));
        fprintf(stderr, "[tb200 run] %zu layers, %d launches, chunks %d, shards %zu, flags %d\n", g->layers.size(), g->num_launches, g->chunks, g->shards.size() + 1, g->flags);
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
    int n = g->num_launches;
    for (tb200_graph* sh : g->shards) n += sh->num_launches;
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
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        const TensorInfo& t = sh->tensors[tensor_id];
        uint8_t* tmp = nullptr;
        CUDA_OK(cudaMalloc(&tmp, t.nchw_bytes));
        cudaError_t e = launch_nhwc_to_nchw(t.dev, tmp, t.d.dims[0], t.d.dims[1], t.d.dims[2], t.d.dims[3], sh->ctx->stream);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync((uint8_t*)host_nchw + (size_t)sh->first_image * image_bytes(sh, tensor_id), tmp, t.nchw_bytes, cudaMemcpyDeviceToHost, sh->ctx->stream);
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
    for (const Step& s : g->steps)
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

// Tables of the per-byte functions of the example's post-processing, with its own arithmetic: dequantisation
// ((float)q - zp) * scale (tm_yolov3_tiny_uint8.cpp:471-478), sigmoid = (float)(1.f / (1.f + exp(-x))) with the C library's double
// exp() (:46-49), and exp(x) kept in double because `float pred_w = exp(dw) * anchor_w` multiplies before narrowing (:230).
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

int tb200_graph_yolo_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts)
{
    if (!g || !p || !out || !counts || max_per_image < 1 || p->num_heads < 1 || p->num_heads > 3) return fail(TB200_ERR_INVALID, "bad arguments");
    const int max_cand = p->max_candidates > 0 ? p->max_candidates : 4096;
    static_assert(sizeof(YoloDet) == sizeof(tb200_detection), "detection record layout");
    const int rc = for_each_shard(g, [&](tb200_graph* sh, int) -> int {
        CUDA_OK(cudaSetDevice(sh->ctx->device));
        cudaStream_t st = sh->ctx->stream;
        const int n_img = sh->num_images;
        YoloCand *cand = nullptr, *sorted = nullptr;
        YoloDet* det = nullptr;
        int *cnt = nullptr, *ocnt = nullptr;
        float* sig = nullptr;
        double* ex = nullptr;
        auto cleanup = [&]() { cudaFree(cand), cudaFree(sorted), cudaFree(det), cudaFree(cnt), cudaFree(ocnt), cudaFree(sig), cudaFree(ex); };
        cudaError_t e = cudaMalloc(&cand, sizeof(YoloCand) * (size_t)n_img * max_cand);
        if (e == cudaSuccess) e = cudaMalloc(&sorted, sizeof(YoloCand) * (size_t)n_img * max_cand);
        if (e == cudaSuccess) e = cudaMalloc(&det, sizeof(YoloDet) * (size_t)n_img * max_per_image);
        if (e == cudaSuccess) e = cudaMalloc(&cnt, sizeof(int) * n_img);
        if (e == cudaSuccess) e = cudaMalloc(&ocnt, sizeof(int) * n_img);
        if (e == cudaSuccess) e = cudaMalloc(&sig, sizeof(float) * 256 * 3);
        if (e == cudaSuccess) e = cudaMalloc(&ex, sizeof(double) * 256 * 3);
        if (e == cudaSuccess) e = cudaMemsetAsync(cnt, 0, sizeof(int) * n_img, st);
        unsigned key_base = 0;
        for (int hd = 0; hd < p->num_heads && e == cudaSuccess; hd++)
        {
            const tb200_yolo_head& H = p->heads[hd];
            if (H.output_index < 0 || H.output_index >= (int)sh->output_ids.size())
            {
                cleanup();
                return fail(TB200_ERR_INVALID, "yolo head %d: output index %d", hd, H.output_index);
            }
            const TensorInfo& t = sh->tensors[sh->output_ids[H.output_index]];
            if (t.d.dims[1] != 3 * (p->num_classes + 5))
            {
                cleanup();
                return fail(TB200_ERR_INVALID, "yolo head %d: %d channels, expected 3 x (5 + %d)", hd, t.d.dims[1], p->num_classes);
            }
            float hs[256];
            double he[256];
            build_yolo_tables(t.d, hs, he);
            e = cudaMemcpyAsync(sig + hd * 256, hs, sizeof hs, cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) e = cudaMemcpyAsync(ex + hd * 256, he, sizeof he, cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st); // hs / he live on this stack frame
            if (e == cudaSuccess)
                e = launch_yolo_decode(t.dev, t.cp, t.d.dims[2], t.d.dims[3], n_img, 3, p->num_classes, sig + hd * 256, ex + hd * 256, (float)H.stride, H.anchors,
                                       p->prob_threshold, cand, cnt, max_cand, key_base, t.d.data_type == TB200_DT_UINT8, st);
            key_base += (unsigned)(t.d.dims[2] * t.d.dims[3] * 3);
        }
        if (e == cudaSuccess) e = launch_yolo_nms(cand, cnt, n_img, max_cand, p->nms_threshold, sorted, det, max_per_image, ocnt, st);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(out + (size_t)sh->first_image * max_per_image, det, sizeof(YoloDet) * (size_t)n_img * max_per_image, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(counts + sh->first_image, ocnt, sizeof(int) * n_img, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        cleanup();
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "yolo_detect: %s", cudaGetErrorString(e));
        return 0;
    });
    cudaSetDevice(g->ctx->device);
    return rc;
}

int tb200_graph_work(tb200_graph* g, double* ops, double* bytes)
{
    if (!g) return fail(TB200_ERR_INVALID, "null graph");
    double o = g->work_ops, b = g->work_bytes;
    for (tb200_graph* sh : g->shards) o += sh->work_ops, b += sh->work_bytes - sh->work_wbytes; // weights count once per launch
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
    int rc = gemm_plan_create(&plan, in, k_pad, weight, out, m, k_pad, oc, cpad(oc), cpad(oc), 0, 0);
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

} // extern "C"
