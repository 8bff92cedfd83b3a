// fl_runtime.cu -- library state, memory, lookup tables and the extern "C" entry points of
// include/fl_cuda.h.  No CPU compute path exists here: every entry point either runs the sm_90a
// kernels or fails loudly.
#include <cuda_fp16.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "fl_common.cuh"
#include "fl_decode.h"
#include "fl_kernels.h"

// ---------------------------------------------------------------------------------------------
// state
// ---------------------------------------------------------------------------------------------
namespace {
struct Scratch {
    void *p = nullptr;
    size_t cap = 0;
};
struct State {
    bool ready = false;
    int device = -1;
    cudaStream_t stream = nullptr;
    uint16_t *tab_silu = nullptr;   // fp16 -> fp16 silu table (device)
    uint16_t *tab_exp = nullptr;    // fp16 -> fp16 exp table (device)
    // cos/sin tables, one per head dimension: [pos][dims/2] for positions [0, pos)
    struct Rope { int dims = 0, pos = 0; float2 *cs = nullptr; };
    std::vector<Rope> rope;
    // Tables replaced by a larger one.  Programs and captured graphs of earlier decode plans still hold their addresses, so they stay
    // allocated until fl_shutdown; capacity doubles on growth, so they add up to less than the live table of their head dimension.
    std::vector<float2 *> rope_retired;
    Scratch scratch[4];
    uint64_t launches = 0;
};
State g;
thread_local char g_err[1024] = "";
// fl_init / fl_shutdown may race when several host threads reach the library first at once.
std::mutex g_init_mu;
// The host-buffer entry points share the scratch slots: a larger request frees and reallocates a
// slot, and every call stages its inputs there.  One caller at a time, from scratch_get to the
// final stream synchronise; they all run on the one library stream anyway, so nothing is lost.
std::mutex g_host_mu;
}  // namespace

void fl_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    if (getenv("FASTLLAMA_B200_VERBOSE")) fprintf(stderr, "[fl_cuda] error: %s\n", g_err);
}
void fl_count_launch() { g.launches++; }

#define FL_NEED_INIT()                                                                               \
    do {                                                                                             \
        if (!g.ready) {                                                                              \
            fl_set_error("libfl_cuda is not initialised (fl_init failed or was never called; there " \
                         "is no CPU fallback)");                                                     \
            return -3;                                                                               \
        }                                                                                            \
    } while (0)

static int scratch_get(int i, size_t bytes, void **out) {
    Scratch &s = g.scratch[i];
    if (s.cap < bytes) {
        if (s.p) FL_CUDA_OK(cudaFree(s.p));
        s.p = nullptr;
        s.cap = 0;
        size_t cap = (bytes + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
        FL_CUDA_OK(cudaMalloc(&s.p, cap));
        s.cap = cap;
    }
    *out = s.p;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// fp16 lookup tables, built exactly like the reference builds them on first ggml_init
// (reference lib/ggml.c:3676-3688): f = fp16->fp32(i); silu = f/(1+expf(-f)); exp = expf(f);
// both rounded to fp16 (round-to-nearest-even).  Host libm, so table contents equal the
// reference's on the same machine.
// ---------------------------------------------------------------------------------------------
static int build_tables() {
    std::vector<uint16_t> silu(1 << 16), ex(1 << 16);
    for (int i = 0; i < (1 << 16); i++) {
        const float f = __half2float(__ushort_as_half((unsigned short)i));
        const float sv = f / (1.0f + expf(-f));
        const float ev = expf(f);
        silu[i] = __half_as_ushort(__float2half_rn(sv));
        ex[i] = __half_as_ushort(__float2half_rn(ev));
    }
    FL_CUDA_OK(cudaMalloc((void **)&g.tab_silu, sizeof(uint16_t) << 16));
    FL_CUDA_OK(cudaMalloc((void **)&g.tab_exp, sizeof(uint16_t) << 16));
    FL_CUDA_OK(cudaMemcpy(g.tab_silu, silu.data(), sizeof(uint16_t) << 16, cudaMemcpyHostToDevice));
    FL_CUDA_OK(cudaMemcpy(g.tab_exp, ex.data(), sizeof(uint16_t) << 16, cudaMemcpyHostToDevice));
    return 0;
}

// rope cos/sin for absolute positions, computed with the reference's recurrence
// (reference lib/ggml.c:8655-8668): theta_0 = (float)pos, theta_{i+1} = theta_i * powf(10000, -2/n_dims)
static State::Rope *rope_of(int n_dims) {
    for (auto &r : g.rope)
        if (r.dims == n_dims) return &r;
    return nullptr;
}
static int ensure_rope(int n_dims, int n_pos) {
    State::Rope *r = rope_of(n_dims);
    if (r && r->pos >= n_pos) return 0;
    int cap = n_pos < 512 ? 512 : n_pos;
    if (r && cap < 2 * r->pos) cap = 2 * r->pos;
    const int half = n_dims / 2;
    std::vector<float2> cs((size_t)cap * half);
    const float theta_scale = powf(10000.0, -2.0f / n_dims);
    for (int p = 0; p < cap; p++) {
        float theta = (float)p;
        for (int i = 0; i < half; i++) {
            cs[(size_t)p * half + i] = make_float2(cosf(theta), sinf(theta));
            theta *= theta_scale;
        }
    }
    float2 *d = nullptr;
    FL_CUDA_OK(cudaMalloc((void **)&d, cs.size() * sizeof(float2)));
    FL_CUDA_OK(cudaMemcpy(d, cs.data(), cs.size() * sizeof(float2), cudaMemcpyHostToDevice));
    if (!r) {
        g.rope.push_back(State::Rope());
        r = &g.rope.back();
    } else {
        g.rope_retired.push_back(r->cs);
    }
    r->dims = n_dims;
    r->pos = cap;
    r->cs = d;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// lifetime
// ---------------------------------------------------------------------------------------------
extern "C" int fl_init(int device) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    if (g.ready) return 0;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        fl_set_error("fl_init: no CUDA device visible (%s); this backend has no CPU fallback",
                     e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
        return -1;
    }
    if (device < 0) {
        const char *env = getenv("FASTLLAMA_DEVICE");
        if (!env) env = getenv("LOCAL_RANK");
        device = env ? atoi(env) : 0;
    }
    FL_REQUIRE(device < count, "fl_init: device %d requested but only %d visible", device, count);
    FL_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    FL_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    FL_REQUIRE(prop.major == 9 && prop.minor == 0, "fl_init: built for sm_90a only, device %d is sm_%d%d (%s)", device, prop.major,
               prop.minor, prop.name);
    FL_CUDA_OK(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
    g.device = device;
    if (flk_query_device() != 0) return -1;
    if (build_tables() != 0) return -1;
    g.ready = true;
    return 0;
}

extern "C" void fl_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    std::lock_guard<std::mutex> lk_host(g_host_mu);
    if (!g.ready) return;
    cudaStreamSynchronize(g.stream);
    for (auto &s : g.scratch) {
        if (s.p) cudaFree(s.p);
        s = Scratch();
    }
    if (g.tab_silu) cudaFree(g.tab_silu);
    if (g.tab_exp) cudaFree(g.tab_exp);
    for (auto &r : g.rope) cudaFree(r.cs);
    for (float2 *p : g.rope_retired) cudaFree(p);
    flk_exact_release();
    cudaStreamDestroy(g.stream);
    g = State();
}

extern "C" int fl_is_initialized(void) { return g.ready ? 1 : 0; }
extern "C" const char *fl_last_error(void) { return g_err; }
extern "C" void *fl_stream(void) { return (void *)g.stream; }
extern "C" uint64_t fl_launch_count(void) { return g.launches; }

extern "C" int fl_device_props(char *name, int name_len, int *sm_count, size_t *hbm_bytes, int *cc_major, int *cc_minor) {
    FL_NEED_INIT();
    cudaDeviceProp prop;
    FL_CUDA_OK(cudaGetDeviceProperties(&prop, g.device));
    if (name && name_len > 0) {
        strncpy(name, prop.name, (size_t)name_len - 1);
        name[name_len - 1] = 0;
    }
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (hbm_bytes) *hbm_bytes = prop.totalGlobalMem;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// memory
// ---------------------------------------------------------------------------------------------
extern "C" void *fl_dev_malloc(size_t bytes) {
    if (!g.ready) {
        fl_set_error("fl_dev_malloc: not initialised");
        return nullptr;
    }
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
    if (e != cudaSuccess) {
        fl_set_error("fl_dev_malloc(%zu): %s", bytes, cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}
extern "C" int fl_dev_free(void *p) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    FL_CUDA_OK(cudaFree(p));
    return 0;
}
extern "C" int fl_dev_memset(void *p, int value, size_t bytes) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaMemsetAsync(p, value, bytes, g.stream));
    return 0;
}
extern "C" int fl_h2d(void *dst, const void *src, size_t bytes) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, g.stream));
    return 0;
}
extern "C" int fl_d2h(void *dst, const void *src, size_t bytes) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, g.stream));
    return 0;
}
extern "C" int fl_d2d(void *dst, const void *src, size_t bytes) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, g.stream));
    return 0;
}
extern "C" int fl_d2d_2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height) {
    FL_NEED_INIT();
    if (width == 0 || height == 0) return 0;
    FL_CUDA_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToDevice, g.stream));
    return 0;
}
extern "C" int fl_sync(void) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}
extern "C" void *fl_host_alloc_pinned(size_t bytes) {
    void *p = nullptr;
    cudaError_t e = cudaMallocHost(&p, bytes ? bytes : 1);
    if (e != cudaSuccess) {
        fl_set_error("fl_host_alloc_pinned(%zu): %s", bytes, cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}
extern "C" int fl_host_free_pinned(void *p) {
    FL_CUDA_OK(cudaFreeHost(p));
    return 0;
}

// ---------------------------------------------------------------------------------------------
// device-resident entry points
// ---------------------------------------------------------------------------------------------
extern "C" int fl_dev_quantize_q8_0(const float *x, size_t x_row_stride_bytes, void *y, int k, int nrows) {
    FL_NEED_INIT();
    return flk_quantize_q8_0(g.stream, x, x_row_stride_bytes, y, k, nrows);
}
extern "C" int fl_dev_mul_mat_q(int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst,
                                size_t drs, int impl) {
    FL_NEED_INIT();
    return flk_mul_mat_q(g.stream, type, W, wrs, M, K, Yq8, N, dst, drs, impl);
}
extern "C" int fl_dev_dequantize_rows(int type, const void *W, size_t wrs, int K, const int32_t *ids, int n_ids,
                                      float *dst, size_t drs) {
    FL_NEED_INIT();
    return flk_dequantize_rows(g.stream, type, W, wrs, K, ids, n_ids, dst, drs);
}
extern "C" int fl_dev_quantize_q4(int type, const float *x, void *y, int k, int nrows) {
    FL_NEED_INIT();
    return flk_quantize_q4(g.stream, type, x, y, k, nrows);
}

extern "C" int fl_dev_quantize_q4_file(int type, int src_type, const void *x, void *y, int k, int nrows, unsigned long long *hist) {
    FL_NEED_INIT();
    FL_REQUIRE(x && y, "fl_dev_quantize_q4_file: null buffer");
    return flk_quantize_q4_file(g.stream, type, src_type, x, y, k, nrows, hist);
}
extern "C" int fl_dev_quantize_q4_file_lora(int type, int src_type, const void *x, int delta_type, const void *delta, void *y, int k, int nrows,
                                            unsigned long long *hist) {
    FL_NEED_INIT();
    FL_REQUIRE(x && y, "fl_dev_quantize_q4_file_lora: null buffer");
    return flk_quantize_q4_file_lora(g.stream, type, src_type, x, delta_type, delta, y, k, nrows, hist);
}

extern "C" int fl_dev_quantize_q4_simd(int type, const float *x, void *y, int k, int nrows) {
    FL_NEED_INIT();
    return flk_quantize_q4_simd(g.stream, type, x, y, k, nrows);
}
extern "C" int fl_dev_add_q_f32(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const float *X, size_t x_row_stride_elems, void *dst,
                                size_t dst_row_stride_bytes) {
    FL_NEED_INIT();
    return flk_add_q_f32(g.stream, type, W, w_row_stride_bytes, M, K, X, x_row_stride_elems, dst, dst_row_stride_bytes);
}
extern "C" int fl_dev_add_q_f16(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const uint16_t *X, size_t x_row_stride_elems, void *dst,
                                size_t dst_row_stride_bytes) {
    FL_NEED_INIT();
    return flk_add_q_f16(g.stream, type, W, w_row_stride_bytes, M, K, X, x_row_stride_elems, dst, dst_row_stride_bytes);
}
extern "C" int fl_dev_scale_f16(const fl_view *t, float v) {
    FL_NEED_INIT();
    int64_t n = 1, nb = 2;
    for (int i = 0; i < 4; i++) {
        FL_REQUIRE(t->nb[i] == nb, "fl_dev_scale_f16: the tensor is not contiguous f16 (nb[%d] = %lld)", i, (long long)t->nb[i]);
        nb *= t->ne[i];
        n *= t->ne[i];
    }
    return flk_scale_f16(g.stream, (uint16_t *)t->data, (long)n, v);
}
extern "C" int fl_dev_mul_mat_f32_ref(const float *A, size_t lda, int Ma, const float *B, size_t ldb, int Mb, int K, float *out, size_t ldo) {
    FL_NEED_INIT();
    return flk_mul_mat_f32_ref(g.stream, A, lda, Ma, B, ldb, Mb, K, out, ldo);
}

extern "C" int fl_dev_rms_norm(const fl_view *src, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_rms_norm(g.stream, *src, *dst, 1e-6f);
}
extern "C" int fl_dev_add(const fl_view *a, const fl_view *b, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_binary(g.stream, FLK_ADD, *a, *b, *dst);
}
extern "C" int fl_dev_mul(const fl_view *a, const fl_view *b, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_binary(g.stream, FLK_MUL, *a, *b, *dst);
}
extern "C" int fl_dev_repeat(const fl_view *src, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_repeat(g.stream, *src, *dst);
}
extern "C" int fl_dev_scale(const fl_view *t, float v) {
    FL_NEED_INIT();
    return flk_scale(g.stream, *t, v);
}
extern "C" int fl_dev_silu(const fl_view *src, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_silu(g.stream, *src, *dst, g.tab_silu);
}
extern "C" int fl_dev_diag_mask_inf(const fl_view *t, int n_past) {
    FL_NEED_INIT();
    return flk_diag_mask_inf(g.stream, *t, n_past);
}
extern "C" int fl_dev_soft_max(const fl_view *t) {
    FL_NEED_INIT();
    return flk_soft_max(g.stream, *t, g.tab_exp);
}
extern "C" int fl_dev_rope(const fl_view *t, int n_past, int n_dims, int mode) {
    FL_NEED_INIT();
    const int need = (int)(((mode & 1) ? 0 : n_past) + t->ne[2]);
    if (ensure_rope(n_dims, need) != 0) return -1;
    const State::Rope *r = rope_of(n_dims);
    return flk_rope(g.stream, *t, n_past, n_dims, mode, r->cs, r->pos);
}
extern "C" int fl_dev_cpy_f32(const fl_view *src, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_cpy_f32(g.stream, *src, *dst);
}
extern "C" int fl_dev_mul_mat_f32(const fl_view *src0, const fl_view *src1, const fl_view *dst) {
    FL_NEED_INIT();
    return flk_mul_mat_f32(g.stream, *src0, *src1, *dst);
}
extern "C" int fl_dev_tp_unshard(const float *gathered, int world, int N, int n_local, const float *residual, float *dst) {
    FL_NEED_INIT();
    return flk_tp_unshard(g.stream, gathered, world, N, n_local, residual, dst);
}
extern "C" int fl_dev_tp_unshard_v(const float *gathered, int world, int N, int slice_stride, const int *first, const int *count, const float *residual,
                                   float *dst) {
    FL_NEED_INIT();
    return flk_tp_unshard_v(g.stream, gathered, world, N, slice_stride, first, count, residual, dst);
}

// ---- fused decode step ------------------------------------------------------------------------
extern "C" int fl_dev_mv_fused_supported(int type, int K, int mtot) { return flk_mv_fused_supported(type, K, mtot); }
extern "C" int fl_dev_rope_table(int n_dims, int n_pos) {
    FL_NEED_INIT();
    return ensure_rope(n_dims, n_pos);
}
extern "C" int fl_dev_mv_fused(const fl_mv_args *args) {
    FL_NEED_INIT();
    fl_mv_args a = *args;
    FL_REQUIRE(a.n_dst_peer == 0 && !a.x_ll && !a.out_ll && !a.res_ll, "fl_dev_mv_fused: dataflow (LL) vectors and peer outputs exist only inside the token kernel");
    a.silu_tab = g.tab_silu;
    if (a.epi == FL_EPI_QKV) {
        const State::Rope *r = rope_of(a.head_dim);
        FL_REQUIRE(r && r->pos >= a.n_ctx, "fl_dev_mv_fused: call fl_dev_rope_table(head_dim, n_ctx) first");
        a.rope_cs = r->cs;
    }
    return flk_mv_fused(g.stream, &a);
}
extern "C" int fl_dev_attn_decode(const float *q, const float *kcache, const float *vcache, float *out, const int *n_past,
                                  int k_row_stride, int n_head, int head_dim, int n_ctx, float scale) {
    FL_NEED_INIT();
    return flk_attn_decode(g.stream, q, kcache, vcache, out, n_past, k_row_stride, n_head, head_dim, n_ctx, scale, g.tab_exp);
}
extern "C" int fl_token_plan_create(const fl_token_step *steps, int n_steps, void **plan_out) { return fl_token_plan_create_ll(steps, n_steps, nullptr, plan_out); }
extern "C" int fl_token_plan_create_ll(const fl_token_step *steps, int n_steps, unsigned *epoch_counter, void **plan_out) {
    FL_NEED_INIT();
    FL_REQUIRE(steps && n_steps > 0 && plan_out, "fl_token_plan_create: bad arguments");
    const State::Rope *rope = nullptr;
    for (int i = 0; i < n_steps; i++)
        if (steps[i].kind == 0 && steps[i].mv.epi == FL_EPI_QKV) {
            const State::Rope *r = rope_of(steps[i].mv.head_dim);
            FL_REQUIRE(r && r->pos >= steps[i].mv.n_ctx && (!rope || rope == r), "fl_token_plan_create: call fl_dev_rope_table(head_dim, n_ctx) first");
            rope = r;
        }
    return flk_token_plan_create(steps, n_steps, g.tab_silu, g.tab_exp, rope ? rope->cs : nullptr, epoch_counter, plan_out);
}
extern "C" int fl_token_plan_launch(void *plan) {
    FL_NEED_INIT();
    return flk_token_plan_launch(g.stream, plan);
}
extern "C" int fl_token_plan_profile(void *plan, unsigned long long *out, size_t max_words, int *n_ctas) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return flk_token_plan_profile(plan, out, max_words, n_ctas);
}
extern "C" int fl_token_plan_profile2(void *plan, unsigned *out, size_t max_words) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return flk_token_plan_profile2(plan, out, max_words);
}
extern "C" int fl_token_plan_error(void *plan) {
    FL_NEED_INIT();
    return flk_token_plan_error(plan);
}
extern "C" int fl_token_plan_destroy(void *plan) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return flk_token_plan_destroy(plan);
}
// ---- tensor parallelism: K-slice packing + NCCL through dlopen ------------------------------------
__global__ void k_pack_cols(const uint32_t *__restrict__ W, size_t src_stride_w, int M, size_t src_off_w, int words, uint32_t *__restrict__ dst,
                            size_t dst_stride_w) {
    const long total = (long)M * words;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long m = i / words, w = i % words;
        dst[m * dst_stride_w + w] = W[m * src_stride_w + src_off_w + w];
    }
}
extern "C" int fl_dev_pack_cols(int type, const void *W, size_t wrs, int M, int blk0, int nblk, void *dst, size_t drs) {
    FL_NEED_INIT();
    const int bb = fl_block_bytes(type);
    FL_REQUIRE(bb > 0 && wrs % 4 == 0 && drs % 4 == 0 && drs >= (size_t)nblk * bb, "fl_dev_pack_cols: bad arguments");
    const int words = nblk * bb / 4;
    k_pack_cols<<<flk_sm_count() * 8, 256, 0, g.stream>>>((const uint32_t *)W, wrs / 4, M, (size_t)blk0 * bb / 4, words, (uint32_t *)dst, drs / 4);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

struct NcclId { char internal[128]; };
namespace {
struct NcclApi {
    void *lib = nullptr;
    void *comm = nullptr;
    int rank = 0, world = 1;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, NcclId, int) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
};
}  // namespace
static NcclApi g_nccl;

static int nccl_load() {
    if (g_nccl.lib) return 0;
    // the soname resolves to whatever libnccl.so.2 the process already has (torch's bundled one under torchrun) or the system's
    g_nccl.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    FL_REQUIRE(g_nccl.lib != nullptr, "cannot dlopen libnccl.so.2: %s", dlerror());
    *(void **)&g_nccl.GetUniqueId = dlsym(g_nccl.lib, "ncclGetUniqueId");
    *(void **)&g_nccl.CommInitRank = dlsym(g_nccl.lib, "ncclCommInitRank");
    *(void **)&g_nccl.AllReduce = dlsym(g_nccl.lib, "ncclAllReduce");
    *(void **)&g_nccl.AllGather = dlsym(g_nccl.lib, "ncclAllGather");
    *(void **)&g_nccl.GetErrorString = dlsym(g_nccl.lib, "ncclGetErrorString");
    FL_REQUIRE(g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.AllGather, "libnccl.so.2 lacks the expected symbols");
    return 0;
}
#define FL_NCCL_OK(expr)                                                                                  \
    do {                                                                                                  \
        int _r = (expr);                                                                                  \
        if (_r != 0) {                                                                                    \
            fl_set_error("%s -> nccl error %d (%s)", #expr, _r, g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?"); \
            return -1;                                                                                    \
        }                                                                                                 \
    } while (0)
extern "C" int fl_comm_unique_id(void *out128) {
    if (nccl_load()) return -1;
    FL_NCCL_OK(g_nccl.GetUniqueId(out128));
    return 0;
}
extern "C" int fl_comm_init(int rank, int world, const void *id128) {
    FL_NEED_INIT();
    if (world <= 1) { g_nccl.rank = 0; g_nccl.world = 1; return 0; }
    if (nccl_load()) return -1;
    NcclId id;
    memcpy(&id, id128, sizeof(id));
    FL_NCCL_OK(g_nccl.CommInitRank(&g_nccl.comm, world, id, rank));
    g_nccl.rank = rank;
    g_nccl.world = world;
    return 0;
}
extern "C" int fl_comm_rank(void) { return g_nccl.rank; }
extern "C" int fl_comm_world(void) { return g_nccl.world; }
extern "C" int fl_comm_allreduce_f32(float *buf, size_t n) {
    FL_NEED_INIT();
    if (g_nccl.world <= 1) return 0;
    FL_NCCL_OK(g_nccl.AllReduce(buf, buf, n, /*ncclFloat32*/ 7, /*ncclSum*/ 0, g_nccl.comm, g.stream));
    fl_count_launch();
    return 0;
}
extern "C" int fl_comm_allgather_f32(const float *send, float *recv, size_t n_per_rank) {
    FL_NEED_INIT();
    if (g_nccl.world <= 1) {
        if (send != recv) FL_CUDA_OK(cudaMemcpyAsync(recv, send, n_per_rank * sizeof(float), cudaMemcpyDeviceToDevice, g.stream));
        return 0;
    }
    FL_NCCL_OK(g_nccl.AllGather(send, recv, n_per_rank, /*ncclFloat32*/ 7, g_nccl.comm, g.stream));
    fl_count_launch();
    return 0;
}

// ---- peer-mapped scratch (CUDA IPC over the NCCL communicator) for collectives fused into the token kernel ----
struct fl_shared_comm {
    void *peers[8] = {nullptr};
    size_t bytes = 0;
    bool ready = false;
};
static fl_shared_comm g_shared;
const void *const *fl_shared_peers(int *rank, int *world) {          // used by fl_token_kernel.cu
    *rank = g_nccl.rank;
    *world = g_nccl.world;
    return g_shared.ready ? (const void *const *)g_shared.peers : nullptr;
}
extern "C" int fl_comm_shared_alloc(size_t bytes, void **peers_out) {
    FL_NEED_INIT();
    const int world = g_nccl.world, rank = g_nccl.rank;
    FL_REQUIRE(world > 1 && world <= 8 && g_nccl.comm, "fl_comm_shared_alloc: needs an initialised communicator of 2..8 ranks");
    FL_REQUIRE(bytes >= 4096, "fl_comm_shared_alloc: the first 4096 bytes are reserved for barrier flags");
    if (g_shared.ready) {
        FL_REQUIRE(bytes <= g_shared.bytes, "fl_comm_shared_alloc: already allocated with %zu bytes", g_shared.bytes);
        for (int r = 0; r < world; r++) peers_out[r] = g_shared.peers[r];
        return 0;
    }
    void *local = nullptr;
    FL_CUDA_OK(cudaMalloc(&local, bytes));
    FL_CUDA_OK(cudaMemset(local, 0, bytes));
    cudaIpcMemHandle_t mine;
    FL_CUDA_OK(cudaIpcGetMemHandle(&mine, local));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    char *d_all = nullptr;
    FL_CUDA_OK(cudaMalloc((void **)&d_all, 64 * (size_t)(world + 1)));
    FL_CUDA_OK(cudaMemcpyAsync(d_all + 64 * (size_t)world, &mine, 64, cudaMemcpyHostToDevice, g.stream));
    FL_NCCL_OK(g_nccl.AllGather(d_all + 64 * (size_t)world, d_all, 16, /*ncclFloat32*/ 7, g_nccl.comm, g.stream));
    cudaIpcMemHandle_t all[8];
    FL_CUDA_OK(cudaMemcpyAsync(all, d_all, 64 * (size_t)world, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    cudaFree(d_all);
    int ok = 1;
    for (int r = 0; r < world; r++) {
        if (r == rank) { g_shared.peers[r] = local; continue; }
        void *p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            fl_set_error("fl_comm_shared_alloc: cudaIpcOpenMemHandle(rank %d) -> %s", r, cudaGetErrorString(e));
            (void)cudaGetLastError();
            ok = 0;
            break;
        }
        g_shared.peers[r] = p;
    }
    // every rank must agree, or some would wait inside the kernel for peers that took the NCCL path
    float *d_ok = nullptr;
    FL_CUDA_OK(cudaMalloc((void **)&d_ok, sizeof(float)));
    const float okf = ok ? 0.f : 1.f;
    FL_CUDA_OK(cudaMemcpyAsync(d_ok, &okf, sizeof(float), cudaMemcpyHostToDevice, g.stream));
    FL_NCCL_OK(g_nccl.AllReduce(d_ok, d_ok, 1, /*ncclFloat32*/ 7, /*ncclSum*/ 0, g_nccl.comm, g.stream));
    float bad = 0.f;
    FL_CUDA_OK(cudaMemcpyAsync(&bad, d_ok, sizeof(float), cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    cudaFree(d_ok);
    if (bad != 0.f) {
        if (ok) fl_set_error("fl_comm_shared_alloc: a peer could not map the shared buffers");
        return -1;
    }
    g_shared.bytes = bytes;
    g_shared.ready = true;
    for (int r = 0; r < world; r++) peers_out[r] = g_shared.peers[r];
    return 0;
}

// a captured graph remembers how many of our kernels it holds, so replays keep fl_launch_count honest
struct fl_graph_handle { cudaGraphExec_t exec; uint64_t kernels; };
static uint64_t g_capture_start = 0;
extern "C" int fl_graph_begin_capture(void) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaStreamBeginCapture(g.stream, cudaStreamCaptureModeThreadLocal));
    g_capture_start = g.launches;
    return 0;
}
extern "C" int fl_graph_end_capture(void **graph_exec_out) {
    FL_NEED_INIT();
    cudaGraph_t graph = nullptr;
    FL_CUDA_OK(cudaStreamEndCapture(g.stream, &graph));
    cudaGraphExec_t exec = nullptr;
    cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
        fl_set_error("cudaGraphInstantiate: %s", cudaGetErrorString(e));
        return -1;
    }
    fl_graph_handle *h = new fl_graph_handle{exec, g.launches - g_capture_start};
    g.launches = g_capture_start;                 // recorded, not executed
    *graph_exec_out = (void *)h;
    return 0;
}
extern "C" int fl_graph_launch(void *graph_exec) {
    FL_NEED_INIT();
    fl_graph_handle *h = (fl_graph_handle *)graph_exec;
    FL_CUDA_OK(cudaGraphLaunch(h->exec, g.stream));
    g.launches += h->kernels;
    return 0;
}
extern "C" int fl_graph_destroy(void *graph_exec) {
    fl_graph_handle *h = (fl_graph_handle *)graph_exec;
    if (h) {
        FL_CUDA_OK(cudaGraphExecDestroy(h->exec));
        delete h;
    }
    return 0;
}

extern "C" void *fl_event_create(void) {
    cudaEvent_t e = nullptr;
    if (cudaEventCreate(&e) != cudaSuccess) {
        fl_set_error("fl_event_create failed");
        return nullptr;
    }
    return (void *)e;
}
extern "C" int fl_event_destroy(void *ev) {
    FL_CUDA_OK(cudaEventDestroy((cudaEvent_t)ev));
    return 0;
}
extern "C" int fl_event_record(void *ev) {
    FL_NEED_INIT();
    FL_CUDA_OK(cudaEventRecord((cudaEvent_t)ev, g.stream));
    return 0;
}
extern "C" int fl_event_sync(void *ev) {
    FL_CUDA_OK(cudaEventSynchronize((cudaEvent_t)ev));
    return 0;
}
extern "C" int fl_event_elapsed_ms(void *a, void *b, float *ms) {
    FL_CUDA_OK(cudaEventElapsedTime(ms, (cudaEvent_t)a, (cudaEvent_t)b));
    return 0;
}

// Counter-based Gaussian fill for synthetic model files (tools only): element i depends on (seed, i)
// alone, so the file contents are reproducible on any grid.  splitmix64 -> two uniforms -> Box-Muller.
__device__ __forceinline__ uint64_t fl_splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__global__ void k_fill_normal(float *__restrict__ p, size_t n, uint64_t seed, float std) {
    const size_t npairs = (n + 1) / 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += (size_t)gridDim.x * blockDim.x) {
        const uint64_t h = fl_splitmix64(seed * 0xD1B54A32D192ED03ull + i);
        const float u1 = ((float)(uint32_t)(h >> 40) + 1.0f) * (1.0f / 16777217.0f);     // (0, 1)
        const float u2 = (float)(uint32_t)((h >> 8) & 0xFFFFFFu) * (1.0f / 16777216.0f);  // [0, 1)
        const float r = sqrtf(-2.0f * logf(u1)) * std;
        float sn, cs;
        sincospif(2.0f * u2, &sn, &cs);
        p[2 * i] = r * cs;
        if (2 * i + 1 < n) p[2 * i + 1] = r * sn;
    }
}
extern "C" int fl_dev_fill_normal(float *p, size_t n, uint64_t seed, float std) {
    FL_NEED_INIT();
    if (n == 0) return 0;
    k_fill_normal<<<flk_sm_count() * 8, 256, 0, g.stream>>>(p, n, seed, std);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// L2 "flush" that leaves CLEAN lines behind: reading a buffer larger than L2 evicts the previous
// working set without creating dirty lines whose write-back would compete with the timed kernel.
__global__ void k_flush_l2(const uint4 *__restrict__ p, size_t n16, unsigned *sink) {
    unsigned acc = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = __ldcg(p + i);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x9e3779b9u) *sink = acc;      // practically never; keeps the loads alive
}

// Timing helper.  W may hold `n_copies` identical copies of the matrix, `copy_stride_bytes` apart;
// launch i reads copy i % n_copies, so with n_copies * matrix bytes > L2 every launch streams its
// weights from HBM exactly as in a decode step (where every matrix is read once per token) and no
// flush kernel sits between the timed launches.  Events bracket the whole batch of `iters` launches.
extern "C" int fl_dev_time_mul_mat_q(int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N,
                                     float *dst, size_t drs, int impl, int iters, size_t flush_l2_bytes,
                                     float *ms_per_launch) {
    return fl_dev_time_mul_mat_q_rot(type, W, wrs, M, K, Yq8, N, dst, drs, impl, iters, flush_l2_bytes, 0, 1, ms_per_launch);
}

// plain streaming-read kernel: calibrates what a trivial kernel achieves on the same bytes
__global__ void __launch_bounds__(512) k_stream_read(const uint4 *__restrict__ p, size_t n16, unsigned *sink) {
    unsigned acc = 0;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 a = __ldcs(p + i), b = __ldcs(p + i + stride), c = __ldcs(p + i + 2 * stride), d = __ldcs(p + i + 3 * stride);
        acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
    }
    for (; i < n16; i += stride) {
        const uint4 a = __ldcs(p + i);
        acc ^= a.x ^ a.y ^ a.z ^ a.w;
    }
    if (acc == 0x9e3779b9u) *sink = acc;
}

// mode: 0 = eager launches, 1 = the batch is captured into a CUDA graph and the graph launch is
// timed (no host launch overhead between kernels), 2 = like 1 but with the calibration read kernel
// over the same byte range instead of the matvec.
extern "C" int fl_dev_time_mul_mat_q_rot(int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N,
                                         float *dst, size_t drs, int impl, int iters, size_t flush_l2_bytes,
                                         size_t copy_stride_bytes, int n_copies, float *ms_per_launch) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(iters > 0 && ms_per_launch && n_copies >= 1, "fl_dev_time_mul_mat_q: bad arguments");
    const int mode = impl >> 8;
    impl &= 0xFF;
    void *flush = nullptr;
    if (flush_l2_bytes) {
        if (scratch_get(3, flush_l2_bytes + 256, &flush) != 0) return -1;
    }
    void *sink = nullptr;
    if (scratch_get(2, 256, &sink) != 0) return -1;
    const size_t mat_bytes = (size_t)M * wrs;
    auto launch_all = [&]() -> int {
        for (int i = 0; i < iters; i++) {
            const char *Wi = (const char *)W + (size_t)(i % n_copies) * copy_stride_bytes;
            if (mode == 2) {
                k_stream_read<<<flk_sm_count() * 4, 512, 0, g.stream>>>((const uint4 *)Wi, mat_bytes / 16, (unsigned *)sink);
                fl_count_launch();
            } else {
                const int rc = flk_mul_mat_q(g.stream, type, Wi, wrs, M, K, Yq8, N, dst, drs, impl);
                if (rc) return rc;
            }
        }
        return 0;
    };
    cudaEvent_t e0, e1;
    FL_CUDA_OK(cudaEventCreate(&e0));
    FL_CUDA_OK(cudaEventCreate(&e1));
    int rc = 0;
    float ms = 0.f;
    if (mode == 0) {
        if (flush) k_flush_l2<<<flk_sm_count() * 8, 256, 0, g.stream>>>((const uint4 *)flush, flush_l2_bytes / 16, (unsigned *)((char *)flush + flush_l2_bytes));
        cudaEventRecord(e0, g.stream);
        rc = launch_all();
        cudaEventRecord(e1, g.stream);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
    } else {
        // one eager launch first (sets function attributes outside the capture)
        if (mode != 2) rc = flk_mul_mat_q(g.stream, type, W, wrs, M, K, Yq8, N, dst, drs, impl);
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        if (rc == 0) {
            FL_CUDA_OK(cudaStreamBeginCapture(g.stream, cudaStreamCaptureModeThreadLocal));
            rc = launch_all();
            cudaError_t ce = cudaStreamEndCapture(g.stream, &graph);
            if (rc == 0 && ce != cudaSuccess) { fl_set_error("graph capture failed: %s", cudaGetErrorString(ce)); rc = -1; }
        }
        if (rc == 0) {
            FL_CUDA_OK(cudaGraphInstantiate(&exec, graph, 0));
            FL_CUDA_OK(cudaGraphLaunch(exec, g.stream));          // warm-up pass
            cudaEventRecord(e0, g.stream);
            FL_CUDA_OK(cudaGraphLaunch(exec, g.stream));
            cudaEventRecord(e1, g.stream);
            cudaEventSynchronize(e1);
            cudaEventElapsedTime(&ms, e0, e1);
        }
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (rc != 0) return rc;
    FL_CUDA_OK(cudaGetLastError());
    *ms_per_launch = ms / iters;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// host-buffer entry points: H2D -> kernel -> D2H, result valid on return
// ---------------------------------------------------------------------------------------------
extern "C" int fl_quantize_rows_q8_0(const float *x, void *y, int k, int nrows) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(x && y && k > 0 && k % FL_QK == 0 && nrows >= 0, "fl_quantize_rows_q8_0: bad arguments (k=%d)", k);
    if (nrows == 0) return 0;
    const size_t xin = (size_t)k * nrows * sizeof(float), yout = (size_t)(k / FL_QK) * nrows * sizeof(fl_block_q8_0);
    void *dx, *dy;
    if (scratch_get(0, xin, &dx) || scratch_get(1, yout, &dy)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dx, x, xin, cudaMemcpyHostToDevice, g.stream));
    if (flk_quantize_q8_0(g.stream, (const float *)dx, (size_t)k * sizeof(float), dy, k, nrows)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(y, dy, yout, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}
extern "C" int fl_quantize_row_q8_0(const float *x, void *y, int k) { return fl_quantize_rows_q8_0(x, y, k, 1); }

extern "C" int fl_quantize_rows_q4(int type, const float *x, void *y, int k, int nrows) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(x && y && k > 0 && k % FL_QK == 0 && nrows >= 0, "fl_quantize_rows_q4: bad arguments (k=%d)", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_quantize_rows_q4: unsupported type %d", type);
    if (nrows == 0) return 0;
    const size_t xin = (size_t)k * nrows * sizeof(float), yout = (size_t)(k / FL_QK) * nrows * fl_block_bytes(type);
    void *dx, *dy;
    if (scratch_get(0, xin, &dx) || scratch_get(1, yout, &dy)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dx, x, xin, cudaMemcpyHostToDevice, g.stream));
    if (flk_quantize_q4(g.stream, type, (const float *)dx, dy, k, nrows)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(y, dy, yout, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}

extern "C" int fl_quantize_rows_q4_simd(int type, const float *x, void *y, int k, int nrows) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(x && y && k > 0 && k % FL_QK == 0 && nrows >= 0, "fl_quantize_rows_q4_simd: bad arguments (k=%d)", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_quantize_rows_q4_simd: unsupported type %d", type);
    if (nrows == 0) return 0;
    const size_t xin = (size_t)k * nrows * sizeof(float), yout = (size_t)(k / FL_QK) * nrows * fl_block_bytes(type);
    void *dx, *dy;
    if (scratch_get(0, xin, &dx) || scratch_get(1, yout, &dy)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dx, x, xin, cudaMemcpyHostToDevice, g.stream));
    if (flk_quantize_q4_simd(g.stream, type, (const float *)dx, dy, k, nrows)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(y, dy, yout, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}

extern "C" int fl_dequantize_rows_q4(int type, const void *x, float *y, int k, int nrows) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(x && y && k > 0 && k % FL_QK == 0 && nrows >= 0, "fl_dequantize_rows_q4: bad arguments (k=%d)", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_dequantize_rows_q4: unsupported type %d", type);
    if (nrows == 0) return 0;
    const size_t rb = (size_t)(k / FL_QK) * fl_block_bytes(type);
    const size_t xin = rb * nrows, yout = (size_t)k * nrows * sizeof(float);
    void *dx, *dy;
    if (scratch_get(0, xin, &dx) || scratch_get(1, yout, &dy)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dx, x, xin, cudaMemcpyHostToDevice, g.stream));
    if (flk_dequantize_rows(g.stream, type, dx, rb, k, nullptr, nrows, (float *)dy, (size_t)k)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(y, dy, yout, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}

extern "C" int fl_get_rows_q(int type, int K, int n_ids, const void *W, int n_rows_total, const int32_t *ids, float *dst) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(W && ids && dst && K > 0 && K % FL_QK == 0, "fl_get_rows_q: bad arguments");
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_get_rows_q: unsupported type %d", type);
    for (int i = 0; i < n_ids; i++)
        FL_REQUIRE(ids[i] >= 0 && ids[i] < n_rows_total, "fl_get_rows_q: id %d out of range [0,%d)", ids[i], n_rows_total);
    if (n_ids <= 0) return 0;
    const size_t rb = (size_t)(K / FL_QK) * fl_block_bytes(type);
    void *dw, *di, *dy;
    if (scratch_get(0, rb * n_rows_total, &dw) || scratch_get(1, (size_t)K * n_ids * 4, &dy) ||
        scratch_get(2, (size_t)n_ids * 4, &di))
        return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dw, W, rb * n_rows_total, cudaMemcpyHostToDevice, g.stream));
    FL_CUDA_OK(cudaMemcpyAsync(di, ids, (size_t)n_ids * 4, cudaMemcpyHostToDevice, g.stream));
    if (flk_dequantize_rows(g.stream, type, dw, rb, K, (const int32_t *)di, n_ids, (float *)dy, (size_t)K)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dst, dy, (size_t)K * n_ids * 4, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}

extern "C" int fl_vec_dot_q4_q8(int type, int n, float *s, const void *x, const void *y) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(s && x && y && n > 0 && n % FL_QK == 0, "fl_vec_dot_q4_q8: bad arguments (n=%d)", n);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_vec_dot_q4_q8: unsupported type %d", type);
    const size_t rb = (size_t)(n / FL_QK) * fl_block_bytes(type), qb = (size_t)(n / FL_QK) * sizeof(fl_block_q8_0);
    void *dw, *dq, *dd;
    if (scratch_get(0, rb, &dw) || scratch_get(1, qb, &dq) || scratch_get(2, 16, &dd)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dw, x, rb, cudaMemcpyHostToDevice, g.stream));
    FL_CUDA_OK(cudaMemcpyAsync(dq, y, qb, cudaMemcpyHostToDevice, g.stream));
    if (flk_mul_mat_q(g.stream, type, dw, rb, 1, n, dq, 1, (float *)dd, 1, 0)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(s, dd, sizeof(float), cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}

extern "C" int fl_mul_mat_q_f32(int type, int M, int K, int N, const void *W, const float *X, float *dst) {
    FL_NEED_INIT();
    std::lock_guard<std::mutex> lk(g_host_mu);
    FL_REQUIRE(W && X && dst && M >= 0 && N >= 0, "fl_mul_mat_q_f32: bad arguments");
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "fl_mul_mat_q_f32: K=%d is not a multiple of 32", K);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "fl_mul_mat_q_f32: unsupported weight type %d", type);
    if (M == 0 || N == 0) return 0;
    const size_t rb = (size_t)(K / FL_QK) * fl_block_bytes(type);
    const size_t wb = rb * M, xb = (size_t)K * N * sizeof(float), qb = (size_t)(K / FL_QK) * N * sizeof(fl_block_q8_0),
                 ob = (size_t)M * N * sizeof(float);
    void *dw, *dxq, *dout;
    // scratch 1 holds X (f32) followed by its q8_0 form
    const size_t xb_al = (xb + 255) & ~(size_t)255;
    if (scratch_get(0, wb, &dw) || scratch_get(1, xb_al + qb, &dxq) || scratch_get(2, ob, &dout)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dw, W, wb, cudaMemcpyHostToDevice, g.stream));
    FL_CUDA_OK(cudaMemcpyAsync(dxq, X, xb, cudaMemcpyHostToDevice, g.stream));
    void *dq = (char *)dxq + xb_al;
    // INIT phase of the reference op: every src1 row -> q8_0 (lib/ggml.c:8105-8119)
    if (flk_quantize_q8_0(g.stream, (const float *)dxq, (size_t)K * sizeof(float), dq, K, N)) return -1;
    // COMPUTE phase (lib/ggml.c:8125-8163)
    const char *impl_env = getenv("FASTLLAMA_B200_MATVEC_IMPL");
    const int impl = impl_env ? atoi(impl_env) : 0;
    if (flk_mul_mat_q(g.stream, type, dw, rb, M, K, dq, N, (float *)dout, (size_t)M, impl)) return -1;
    FL_CUDA_OK(cudaMemcpyAsync(dst, dout, ob, cudaMemcpyDeviceToHost, g.stream));
    FL_CUDA_OK(cudaStreamSynchronize(g.stream));
    return 0;
}
