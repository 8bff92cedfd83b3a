// fl_ops_kernels.cu -- the non-quantised ops of the LLaMA eval graph (SURVEY.md section 8 row f1),
// kept on the device so activations never leave HBM between the quantised matmuls.
//
// Semantics follow the reference op for op (citations: reference lib/ggml.c):
//   rms_norm      :7378-7434  sum of fp32 squares accumulated in double, mean -> float,
//                             scale = 1/sqrtf(mean + 1e-6f), y = x*scale
//   add / mul     :6259-6330, :6613-6680   element-wise, same shape
//   repeat        :6912-6960
//   scale         :8209-8250  y *= v
//   silu          :3207-3215, :7241-7280   y = fp16_table_silu[fp16(x)]  (table built on the host)
//   diag_mask_inf :8466-8500
//   soft_max      :8521-8589  p = fp16_table_exp[fp16(x - max)], double sum, y = p * (float)(1/sum)
//   rope          :8609-8697  mode 0 adjacent pairs; cos/sin table built on the host with libm
//   cpy/dup f32   :5942-6257  logical-order element copy between arbitrary strided views
//   mul_mat f32   :7482-7680  dst[i0,i1,i2,i3] = dot(src0 row i0, src1 row i1) per (i2,i3), in ggml_vec_dot_f32's order (fl_exact_kernels.cu)
// rms_norm adds the squares in double in a different order than the reference's scalar loop (the float mean can differ only when
// the double sum sits within ~1e-14 relative of a rounding boundary); soft_max's double sum is EXACT in any order (every term is an
// fp16 value <= 1, i.e. a multiple of 2^-24); everything table-driven is exact.
#include <cuda_fp16.h>

#include <type_traits>

#include "fl_common.cuh"
#include "fl_kernels.h"

static inline int ew_grid(long n, int threads) {
    long g = (n + threads - 1) / threads;
    const long cap = (long)flk_sm_count() * 32;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

__device__ __forceinline__ int64_t fl_off4(const fl_view &v, int64_t i0, int64_t i1, int64_t i2, int64_t i3) {
    return i0 * v.nb[0] + i1 * v.nb[1] + i2 * v.nb[2] + i3 * v.nb[3];
}
// logical linear index -> byte offset
__device__ __forceinline__ int64_t fl_off_lin(const fl_view &v, int64_t n) {
    const int64_t i0 = n % v.ne[0]; n /= v.ne[0];
    const int64_t i1 = n % v.ne[1]; n /= v.ne[1];
    const int64_t i2 = n % v.ne[2];
    const int64_t i3 = n / v.ne[2];
    return fl_off4(v, i0, i1, i2, i3);
}
static inline int64_t nelem(const fl_view &v) { return v.ne[0] * v.ne[1] * v.ne[2] * v.ne[3]; }

// ------------------------------------------------------------------------------------------------
// rms_norm: one CTA (256 threads) per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rms_norm(const fl_view src, const fl_view dst, float eps) {
    const int64_t row = blockIdx.x;
    const int64_t i1 = row % src.ne[1], i2 = (row / src.ne[1]) % src.ne[2], i3 = row / (src.ne[1] * src.ne[2]);
    const float *x = (const float *)((const char *)src.data + fl_off4(src, 0, i1, i2, i3));
    float *y = (float *)((char *)dst.data + fl_off4(dst, 0, i1, i2, i3));
    const int n = (int)src.ne[0];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = x[i];
        acc += (double)__fmul_rn(v, v);
    }
    __shared__ double red[8];
    __shared__ float s_scale;
    acc = fl_warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w];
        const float mean = (float)(t / (double)n);
        s_scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
    }
    __syncthreads();
    const float scale = s_scale;
    for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = __fmul_rn(x[i], scale);
}

int flk_rms_norm(cudaStream_t st, const fl_view &src, const fl_view &dst, float eps) {
    FL_REQUIRE(src.nb[0] == 4 && dst.nb[0] == 4, "rms_norm: rows must be contiguous f32");
    const int64_t rows = src.ne[1] * src.ne[2] * src.ne[3];
    if (rows <= 0) return 0;
    k_rms_norm<<<(unsigned)rows, 256, 0, st>>>(src, dst, eps);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// element-wise binary / repeat / scale / silu
// ------------------------------------------------------------------------------------------------
template <int OP>
__global__ void k_binary(const fl_view a, const fl_view b, const fl_view d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = *(const float *)((const char *)a.data + fl_off_lin(a, i));
        const float y = *(const float *)((const char *)b.data + fl_off_lin(b, i));
        *(float *)((char *)d.data + fl_off_lin(d, i)) = (OP == FLK_ADD) ? __fadd_rn(x, y) : __fmul_rn(x, y);
    }
}
int flk_binary(cudaStream_t st, int op, const fl_view &a, const fl_view &b, const fl_view &dst) {
    const int64_t n = nelem(dst);
    FL_REQUIRE(nelem(a) == n && nelem(b) == n, "binary op: shapes differ");
    if (n <= 0) return 0;
    if (op == FLK_ADD) k_binary<FLK_ADD><<<ew_grid(n, 256), 256, 0, st>>>(a, b, dst, n);
    else               k_binary<FLK_MUL><<<ew_grid(n, 256), 256, 0, st>>>(a, b, dst, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

__global__ void k_repeat(const fl_view s, const fl_view d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i;
        const int64_t i0 = r % d.ne[0]; r /= d.ne[0];
        const int64_t i1 = r % d.ne[1]; r /= d.ne[1];
        const int64_t i2 = r % d.ne[2];
        const int64_t i3 = r / d.ne[2];
        const float v = *(const float *)((const char *)s.data + fl_off4(s, i0 % s.ne[0], i1 % s.ne[1], i2 % s.ne[2], i3 % s.ne[3]));
        *(float *)((char *)d.data + fl_off4(d, i0, i1, i2, i3)) = v;
    }
}
int flk_repeat(cudaStream_t st, const fl_view &src, const fl_view &dst) {
    const int64_t n = nelem(dst);
    if (n <= 0) return 0;
    k_repeat<<<ew_grid(n, 256), 256, 0, st>>>(src, dst, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

__global__ void k_scale(const fl_view t, float v, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float *p = (float *)((char *)t.data + fl_off_lin(t, i));
        *p = __fmul_rn(*p, v);
    }
}
int flk_scale(cudaStream_t st, const fl_view &t, float v) {
    const int64_t n = nelem(t);
    if (n <= 0) return 0;
    k_scale<<<ew_grid(n, 256), 256, 0, st>>>(t, v, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

__global__ void k_silu(const fl_view s, const fl_view d, const uint16_t *__restrict__ tab, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = *(const float *)((const char *)s.data + fl_off_lin(s, i));
        const uint16_t h = __half_as_ushort(__float2half_rn(x));
        *(float *)((char *)d.data + fl_off_lin(d, i)) = __half2float(__ushort_as_half(tab[h]));
    }
}
int flk_silu(cudaStream_t st, const fl_view &src, const fl_view &dst, const uint16_t *tab) {
    const int64_t n = nelem(dst);
    if (n <= 0) return 0;
    k_silu<<<ew_grid(n, 256), 256, 0, st>>>(src, dst, tab, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// diag_mask_inf: element (i, j, k) of [nc, nr, nz] is set to -inf when i > n_past + j
// ------------------------------------------------------------------------------------------------
__global__ void k_diag_mask_inf(const fl_view t, int n_past, int64_t n) {
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx;
        const int64_t i = r % t.ne[0]; r /= t.ne[0];
        const int64_t j = r % t.ne[1];
        const int64_t k = r / t.ne[1];           // ne2*ne3 flattened exactly as the reference (nz = n/nr)
        if (i > n_past + j) *(float *)((char *)t.data + i * t.nb[0] + j * t.nb[1] + k * t.nb[2]) = -INFINITY;
    }
}
int flk_diag_mask_inf(cudaStream_t st, const fl_view &t, int n_past) {
    const int64_t n = nelem(t);
    if (n <= 0) return 0;
    k_diag_mask_inf<<<ew_grid(n, 256), 256, 0, st>>>(t, n_past, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// soft_max over contiguous rows: one warp per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_soft_max(float *__restrict__ data, int nc, int64_t nr, int64_t row_stride_bytes,
                                                  const uint16_t *__restrict__ tab) {
    const int lane = threadIdx.x & 31;
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = wid; r < nr; r += nw) {
        float *p = (float *)((char *)data + r * row_stride_bytes);
        float mx = -INFINITY;
        for (int i = lane; i < nc; i += 32) mx = fmaxf(mx, p[i]);
        mx = fl_warp_max(mx);
        double sum = 0.0;
        for (int i = lane; i < nc; i += 32) {
            const float v = p[i];
            float e = 0.0f;
            if (v != -INFINITY) {
                const uint16_t h = __half_as_ushort(__float2half_rn(__fsub_rn(v, mx)));
                e = __half2float(__ushort_as_half(tab[h]));
                sum += (double)e;
            }
            p[i] = e;
        }
        sum = fl_warp_sum_d(sum);
        const float inv = (float)(1.0 / sum);
        __syncwarp();
        for (int i = lane; i < nc; i += 32) p[i] = __fmul_rn(p[i], inv);
    }
}
int flk_soft_max(cudaStream_t st, const fl_view &t, const uint16_t *tab) {
    FL_REQUIRE(t.nb[0] == 4, "soft_max: rows must be contiguous f32");
    FL_REQUIRE(t.nb[2] == t.nb[1] * t.ne[1] && t.nb[3] == t.nb[2] * t.ne[2], "soft_max: tensor must be contiguous");
    const int64_t nr = t.ne[1] * t.ne[2] * t.ne[3];
    if (nr <= 0) return 0;
    long g = (nr + 7) / 8;
    if (g > (long)flk_sm_count() * 16) g = (long)flk_sm_count() * 16;
    k_soft_max<<<(int)g, 256, 0, st>>>((float *)t.data, (int)t.ne[0], nr, t.nb[1], tab);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// rope, mode 0 (adjacent pairs) and neox (mode & 2); in place.  t = [ne0, ne1(heads), ne2(tokens), ne3]
// ------------------------------------------------------------------------------------------------
__global__ void k_rope(const fl_view t, int n_past, int n_dims, int mode, const float2 *__restrict__ cs, int64_t npairs) {
    const int half = n_dims / 2;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < npairs; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx;
        const int ip = (int)(r % half); r /= half;
        const int64_t i1 = r % t.ne[1]; r /= t.ne[1];
        const int64_t i2 = r % t.ne[2];
        const int64_t i3 = r / t.ne[2];
        if ((mode & 1) && i2 < n_past) continue;
        const int pos = (mode & 1) ? (int)i2 : n_past + (int)i2;
        const float2 c = cs[(size_t)pos * half + ip];
        char *base = (char *)t.data + fl_off4(t, 0, i1, i2, i3);
        float *p0, *p1;
        if (!(mode & 2)) { p0 = (float *)(base + (int64_t)(2 * ip) * t.nb[0]); p1 = (float *)(base + (int64_t)(2 * ip + 1) * t.nb[0]); }
        else             { p0 = (float *)(base + (int64_t)ip * t.nb[0]);       p1 = (float *)(base + (int64_t)(ip + half) * t.nb[0]); }
        const float x0 = *p0, x1 = *p1;
        // reference: x0*cos - x1*sin ; x0*sin + x1*cos (gcc contracts each to one fma in GNU mode)
        *p0 = __fmaf_rn(x0, c.x, -__fmul_rn(x1, c.y));
        *p1 = __fmaf_rn(x0, c.y, __fmul_rn(x1, c.x));
    }
}
int flk_rope(cudaStream_t st, const fl_view &t, int n_past, int n_dims, int mode, const float2 *cs, int n_pos) {
    FL_REQUIRE(n_dims > 0 && n_dims % 2 == 0 && n_dims <= t.ne[0], "rope: bad n_dims %d", n_dims);
    const int64_t max_pos = ((mode & 1) ? 0 : n_past) + t.ne[2];
    FL_REQUIRE(max_pos <= n_pos, "rope: position %lld beyond the cos/sin table (%d)", (long long)max_pos, n_pos);
    const int64_t npairs = (int64_t)(n_dims / 2) * t.ne[1] * t.ne[2] * t.ne[3];
    if (npairs <= 0) return 0;
    k_rope<<<ew_grid(npairs, 256), 256, 0, st>>>(t, n_past, n_dims, mode, cs, npairs);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// cpy f32 -> f32 between strided views (logical element order preserved)
// ------------------------------------------------------------------------------------------------
__global__ void k_cpy_f32(const fl_view s, const fl_view d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        *(float *)((char *)d.data + fl_off_lin(d, i)) = *(const float *)((const char *)s.data + fl_off_lin(s, i));
    }
}
int flk_cpy_f32(cudaStream_t st, const fl_view &src, const fl_view &dst) {
    const int64_t n = nelem(src);
    FL_REQUIRE(n == nelem(dst), "cpy: element counts differ");
    if (n <= 0) return 0;
    k_cpy_f32<<<ew_grid(n, 256), 256, 0, st>>>(src, dst, n);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// tensor-parallel unshard: an all-gather of every rank's [N][n_local] slice leaves [world][N][n_local]; the eval needs
// [N][world * n_local] (rank r's slice = elements [r * n_local, (r + 1) * n_local) of every row), optionally + residual, added
// with one fp32 rounding per element as ggml_add does (reference lib/ggml.c:6259-6330).  V = 4: float4 loads and stores
// (n_local % 4 == 0 and 16-byte aligned buffers), else one float at a time.
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void k_tp_unshard(const float *__restrict__ g, int world, int N, int n_local, const float *res, float *dst) {
    using T = typename std::conditional<V == 4, float4, float>::type;
    const int nlv = n_local / V;
    const int64_t row = (int64_t)world * nlv, n = (int64_t)N * row;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t col = i / row, c = i - col * row;
        const int r = (int)(c / nlv), j = (int)(c - (int64_t)r * nlv);
        T v = ((const T *)g)[((int64_t)r * N + col) * nlv + j];
        if (res) {
            const T b = ((const T *)res)[i];
            if constexpr (V == 4) { v.x = __fadd_rn(v.x, b.x); v.y = __fadd_rn(v.y, b.y); v.z = __fadd_rn(v.z, b.z); v.w = __fadd_rn(v.w, b.w); }
            else v = __fadd_rn(v, b);
        }
        ((T *)dst)[i] = v;
    }
}
int flk_tp_unshard(cudaStream_t st, const float *gathered, int world, int N, int n_local, const float *residual, float *dst) {
    FL_REQUIRE(gathered && dst && world >= 1 && N >= 0 && n_local >= 0, "tp_unshard: bad arguments");
    const int64_t n = (int64_t)N * world * n_local;
    if (n == 0) return 0;
    const bool vec = n_local % 4 == 0 && (((uintptr_t)gathered | (uintptr_t)dst | (uintptr_t)residual) & 15) == 0;
    if (vec) k_tp_unshard<4><<<ew_grid(n / 4, 256), 256, 0, st>>>(gathered, world, N, n_local, residual, dst);
    else     k_tp_unshard<1><<<ew_grid(n, 256), 256, 0, st>>>(gathered, world, N, n_local, residual, dst);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// the same for uneven slices (tensor parallelism at a world size that does not divide the shape): rank r's [N][count_r] block
// sits at g + r * N * stride (the all-gather of slices padded to `stride` floats) and goes to columns [first_r, first_r + count_r)
// of [N][n], n = sum of the counts.  One thread per V consecutive elements of one rank's block row; the per-rank tables are
// kernel parameters.  V = 4 for ranks whose count, first column and block start keep every float4 16-byte aligned (the caller
// checks this per rank, k_vmask); the other ranks are covered by the V = 1 launch.  Each element is written by exactly one launch.
// ------------------------------------------------------------------------------------------------
struct tp_slices {
    int first[8], count[8];
    int64_t start[9];        // prefix sums of N * (count_r / V): thread i belongs to the rank r with start[r] <= i < start[r + 1]
};
template <int V>
__global__ void k_tp_unshard_v(const float *__restrict__ g, int world, int N, int stride, int n, const tp_slices t, const float *res, float *dst) {
    using T = typename std::conditional<V == 4, float4, float>::type;
    const int64_t total = t.start[world];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int r = 0;
        while (i >= t.start[r + 1]) r++;
        const int cv = t.count[r] / V;
        const int64_t k = i - t.start[r], col = k / cv;
        const int j = (int)(k - col * cv) * V;
        T v =*(const T *)(g + (int64_t)r * N * stride + col * t.count[r] + j);
        const int64_t o = col * n + t.first[r] + j;
        if (res) {
            const T b = *(const T *)(res + o);
            if constexpr (V == 4) { v.x = __fadd_rn(v.x, b.x); v.y = __fadd_rn(v.y, b.y); v.z = __fadd_rn(v.z, b.z); v.w = __fadd_rn(v.w, b.w); }
            else v = __fadd_rn(v, b);
        }
        *(T *)(dst + o) = v;
    }
}
int flk_tp_unshard_v(cudaStream_t st, const float *gathered, int world, int N, int stride, const int *first, const int *count, const float *residual,
                     float *dst) {
    FL_REQUIRE(gathered && dst && first && count && world >= 1 && world <= 8 && N >= 0 && stride >= 0, "tp_unshard_v: bad arguments");
    int n = 0;
    for (int r = 0; r < world; r++) {
        FL_REQUIRE(count[r] >= 0 && count[r] <= stride && first[r] >= 0, "tp_unshard_v: rank %d has a bad slice (%d, %d)", r, first[r], count[r]);
        n += count[r];
    }
    for (int r = 0; r < world; r++) FL_REQUIRE((int64_t)first[r] + count[r] <= n, "tp_unshard_v: rank %d's slice ends past the %d columns", r, n);
    if ((int64_t)N * n == 0) return 0;
    // float4 for a rank when its block rows and its output columns stay 16-byte aligned in every row
    const bool base16 = (((uintptr_t)gathered | (uintptr_t)dst | (uintptr_t)residual) & 15) == 0;
    tp_slices t4, t1;
    t4.start[0] = t1.start[0] = 0;
    for (int r = 0; r < world; r++) {
        const bool vec = base16 && count[r] % 4 == 0 && first[r] % 4 == 0 && n % 4 == 0 && ((int64_t)r * N * stride) % 4 == 0;
        t4.first[r] = t1.first[r] = first[r];
        t4.count[r] = vec ? count[r] : 0;
        t1.count[r] = vec ? 0 : count[r];
        t4.start[r + 1] = t4.start[r] + (int64_t)N * (t4.count[r] / 4);
        t1.start[r + 1] = t1.start[r] + (int64_t)N * t1.count[r];
    }
    for (int r = world; r < 8; r++) { t4.first[r] = t1.first[r] = 0; t4.count[r] = t1.count[r] = 0; t4.start[r + 1] = t4.start[world]; t1.start[r + 1] = t1.start[world]; }
    if (t4.start[world] > 0) {
        k_tp_unshard_v<4><<<ew_grid(t4.start[world], 256), 256, 0, st>>>(gathered, world, N, stride, n, t4, residual, dst);
        fl_count_launch();
        FL_CUDA_OK(cudaGetLastError());
    }
    if (t1.start[world] > 0) {
        k_tp_unshard_v<1><<<ew_grid(t1.start[world], 256), 256, 0, st>>>(gathered, world, N, stride, n, t1, residual, dst);
        fl_count_launch();
        FL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// mul_mat f32 x f32 (attention scores and weighted values of a multi-token eval): the reference-order kernel of
// fl_exact_kernels.cu (one warp per output group, lane l = element l of ggml_vec_dot_f32's 32-float step).
// ------------------------------------------------------------------------------------------------
int flk_mul_mat_f32(cudaStream_t st, const fl_view &src0, const fl_view &src1, const fl_view &dst) {
    FL_REQUIRE(src0.ne[0] == src1.ne[0], "mul_mat_f32: inner dimensions differ");
    return flk_mul_mat_f32_ref4(st, src0, src1, dst);
}
