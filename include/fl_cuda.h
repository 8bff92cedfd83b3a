/*
 * fl_cuda.h -- the thin extern-"C" CUDA layer of the H100 backend (libfl_cuda.so).
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary.  Every entry point
 * cites the reference interface it replaces (file:line relative to the reference tree).
 *
 * Two groups:
 *   (1) HOST-BUFFER entry points: drop-in replacements for the row functions the reference
 *       dispatches through quantize_fns[type] (lib/ggml.c:1731-1773, type quantize_fns_t
 *       include/ggml.h:850-862) and for ggml_compute_forward_mul_mat_q_f32.  Inputs and outputs
 *       are host memory; each call does H2D -> sm_90a kernel -> D2H on the library stream and
 *       returns when the result is in the output buffer.  This is what a cgo/ctypes/FFI binding of
 *       the reference's test hook (ggml_internal_get_quantize_fn) would bind.
 *   (2) DEVICE-RESIDENT entry points (fl_dev_*): the same kernels on device pointers, used by the
 *       ggml-compatible graph executor (include/fl_ggml.h) so weights, KV cache and activations
 *       never leave HBM between ops.
 *
 * Conventions: every function returning int returns 0 on success, negative on error
 * (fl_last_error() describes it).  There is no CPU fallback: without a CUDA device fl_init fails
 * and every other entry point fails with "not initialised".  All work is issued on one internal
 * stream.  fl_init and the host-buffer entry points of group (1) may be called from several host
 * threads at once (the reference's quantize tool calls ggml_quantize_chunk from a thread pool,
 * lib/llama.cpp:613-645): one library mutex is held from the staging-buffer lookup to the final
 * stream synchronise, so concurrent calls run one after another.  Everything else expects a
 * single caller thread (the reference drives ggml from one thread, SURVEY.md 8b).
 */
#ifndef FL_CUDA_H
#define FL_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ggml_type values the backend understands (include/ggml.h:201-214; file-format contract) */
enum { FL_F32 = 0, FL_F16 = 1, FL_Q4_0 = 2, FL_Q4_1 = 3, FL_Q8_0 = 6 };

/* ---- lifetime ---------------------------------------------------------------------------- */
int fl_init(int device);              /* idempotent; device = -1 -> $FASTLLAMA_DEVICE or $LOCAL_RANK or 0 */
void fl_shutdown(void);
int fl_is_initialized(void);
const char *fl_last_error(void);
int fl_device_props(char *name, int name_len, int *sm_count, size_t *hbm_bytes, int *cc_major, int *cc_minor);
void *fl_stream(void);                /* the cudaStream_t all launches use (for CUDA-event timing) */

/* ---- (1) host-buffer entry points --------------------------------------------------------- */

/* quantize_row_q8_0 == quantize_fns[Q4_0|Q4_1].quantize_row_q_dot (lib/ggml.c:1299-1441; AVX2
 * semantics: d = amax/127, id = 127/amax, round-half-even, s = d*sum).  x: k floats, y: k/32
 * q8_0 blocks.  Bit-exact with the reference. */
int fl_quantize_row_q8_0(const float *x, void *y, int k);
int fl_quantize_rows_q8_0(const float *x, void *y, int k, int nrows);

/* quantize_row_q4_0_reference / _q4_1_reference == quantize_fns[type].quantize_row_q_reference,
 * the functions that define model-file contents (lib/ggml.c:630-664, :917-956, used by
 * ggml_quantize_q4_0/_q4_1 :12122-12166).  Bit-exact. */
int fl_quantize_rows_q4(int type, const float *x, void *y, int k, int nrows);

/* quantize_row_q4_0 / quantize_row_q4_1 == quantize_fns[type].quantize_row_q, the SIMD quantisers (lib/ggml.c:666-915 AVX2 branch
 * :739-803, :958-1079 AVX2 branch :965-1038): q4_0 uses id = 7/amax and round-half-even, q4_1 round-half-even.  This is what
 * ggml_compute_forward_add_q_f32 (:6516-6518) re-quantises a LoRA-merged row with.  Bit-exact with the reference's x86 build. */
int fl_quantize_rows_q4_simd(int type, const float *x, void *y, int k, int nrows);

/* dequantize_row_q4_0 / _q4_1 == quantize_fns[type].dequantize_row_q (lib/ggml.c:1443-1665).
 * Bit-exact (q4_1 uses a fused multiply-add like the reference's GNU-mode x86 build). */
int fl_dequantize_rows_q4(int type, const void *x, float *y, int k, int nrows);

/* ggml_vec_dot_q4_0_q8_0 / ggml_vec_dot_q4_1_q8_0 == quantize_fns[type].vec_dot_q
 * (lib/ggml.c:2368-2714): *s = sum over k/32 blocks.  Integer block sums exact; fp32
 * accumulation order differs from the AVX2 lanes (tolerance in tests/test_gpu_rowfns.py). */
int fl_vec_dot_q4_q8(int type, int n, float *s, const void *x, const void *y);

/* ggml_compute_forward_mul_mat_q_f32 (lib/ggml.c:7928-8176) on host buffers:
 * W: M rows of K/32 blocks of `type`, X: N rows of K floats, dst: N rows of M floats.
 * INIT phase (q8_0 quantisation of X) + COMPUTE phase both run on the GPU. */
int fl_mul_mat_q_f32(int type, int M, int K, int N, const void *W, const float *X, float *dst);

/* get_rows on a quantized matrix (ggml_compute_forward_get_rows_q, lib/ggml.c:8333-8360) */
int fl_get_rows_q(int type, int K, int n_ids, const void *W, int n_rows_total, const int32_t *ids, float *dst);

/* ---- (2) device-resident entry points ------------------------------------------------------ */
void *fl_dev_malloc(size_t bytes);
int fl_dev_free(void *p);
int fl_dev_memset(void *p, int value, size_t bytes);
int fl_h2d(void *dst_dev, const void *src_host, size_t bytes);   /* async on the library stream */
int fl_d2h(void *dst_host, const void *src_dev, size_t bytes);   /* async; call fl_sync before reading */
int fl_d2d(void *dst_dev, const void *src_dev, size_t bytes);
/* strided device-to-device copy: `height` rows of `width_bytes`, rows `dpitch` / `spitch` bytes apart (async) */
int fl_d2d_2d(void *dst_dev, size_t dpitch, const void *src_dev, size_t spitch, size_t width_bytes, size_t height);
int fl_sync(void);
void *fl_host_alloc_pinned(size_t bytes);
int fl_host_free_pinned(void *p);

/* activations -> q8_0 rows.  x row r starts at x + r*x_row_stride_bytes; y rows are packed. */
int fl_dev_quantize_q8_0(const float *x, size_t x_row_stride_bytes, void *y, int k, int nrows);

/* dst[n*dst_row_stride + m] = vec_dot(W row m, Yq8 row n).  impl: 0 = auto (N = 1: ring; N >= 16: wgmma GEMM; N >= 4: mma.sync kernel;
 * else plain), 1 = plain warp-per-row LDG kernel, 2 = TMA-bulk-staged persistent matvec (N = 1 only), 3 = legacy tensor-core kernel
 * (mma.sync m16n8k32 u8 x s8 block sums, fp32 scales; any N), 4 = wgmma GEMM (fl_umma_kernel.cu: one wgmma M = 64,
 * K = 32 with 8-bit operands per quant block into registers, weights by TMA, exact fp32 block scaling; needs 16-byte aligned W rows),
 * 5 / 6 / 7 = the same with the column tile forced to 32 / 64 / 64, 8 = reference-order kernel (the reference's fp32 order and bits;
 * any N, 4-byte aligned W rows), 9 = the same arithmetic as a shared-memory-tiled GEMM (k_mul_mat_q_ref_tiled; any N, needs 16-byte
 * aligned W and row stride, else an error).  Impl 0 uses 9 for 8..15 columns and, under FASTLLAMA_B200_INGEST=exact, for every N >= 8. */
int fl_dev_mul_mat_q(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const void *Yq8, int N,
                     float *dst, size_t dst_row_stride_elems, int impl);

int fl_dev_dequantize_rows(int type, const void *W, size_t w_row_stride_bytes, int K, const int32_t *ids_dev,
                           int n_ids, float *dst, size_t dst_row_stride_elems);
int fl_dev_quantize_q4(int type, const float *x, void *y, int k, int nrows);

/* Model-file quantisation (the tensor loop of fastllama::quantize, lib/llama.cpp:585-646): nrows rows
 * of k elements as the input file stores them (src_type 0 = f32, 1 = f16; f16 converts exactly like
 * ggml_fp16_to_fp32; 2 = f32 rounded to f16, nearest even, and widened back, the values of an f32
 * checkpoint after the reference converter's f16 step) -> q4_0 / q4_1 blocks with the bits of
 * fl_quantize_rows_q4.  hist_dev (16
 * counters, may be NULL) is incremented by the count of each stored nibble value, the histogram
 * ggml_quantize_chunk reports.  Asynchronous on the library stream, like every fl_dev_* call. */
int fl_dev_quantize_q4_file(int type, int src_type, const void *x_dev, void *y_dev, int k, int nrows,
                            unsigned long long *hist_dev);

/* ---- attach_lora / detach_lora on the device (reference lib/llama.cpp:697-944; SURVEY.md section 8 row f4) ----
 * fl_dev_quantize_q4_simd: device-resident fl_quantize_rows_q4_simd.
 * fl_dev_add_q_f32: ggml_compute_forward_add_q_f32 (lib/ggml.c:6414-6520): row r of dst = quantize_row_q(dequantize_row_q(row r of W) +
 *   row r of X); dst may be W itself (ggml_add_inplace).  Bit-exact.
 * fl_dev_add_q_f16: ggml_compute_forward_add_q_f16 (lib/ggml.c:12372-12483), the merge of a cached f16 adapter: fl_dev_add_q_f32 with X
 *   as f16 bits, each element widened exactly to fp32 before the one fp32 add.  Bit-exact.
 * fl_dev_scale_f16: ggml_compute_forward_scale_f16 (:12485-12524), in place on a contiguous f16 tensor: x = fp16_rn(fp32(x) * v).
 * fl_dev_mul_mat_f32_ref: ggml_mul_mat of two f32 matrices with ggml_vec_dot_f32's summation order of the AVX2 + FMA build
 *   (lib/ggml.c:2295-2325): out[j * ldo + i] = dot(A row i, B row j), K elements.  Bit-exact; meant for small K (B*A of a LoRA adapter). */
int fl_dev_quantize_q4_simd(int type, const float *x, void *y, int k, int nrows);
int fl_dev_add_q_f32(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const float *X, size_t x_row_stride_elems, void *dst,
                     size_t dst_row_stride_bytes);
int fl_dev_add_q_f16(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const uint16_t *X, size_t x_row_stride_elems, void *dst,
                     size_t dst_row_stride_bytes);
int fl_dev_mul_mat_f32_ref(const float *A, size_t lda_elems, int Ma, const float *B, size_t ldb_elems, int Mb, int K, float *out, size_t ldo_elems);

/* Timing helpers for bench.py / profiling (CUDA events on the library stream, mean ms per launch
 * over `iters` back-to-back launches).  W may hold n_copies identical copies of the matrix,
 * copy_stride_bytes apart; launch i reads copy i % n_copies, so with n_copies * bytes > L2 every
 * launch streams its weights from HBM, as in a decode step where each matrix is read once per token.
 * flush_l2_bytes > 0: a buffer of that size is READ once before the timed batch (clean eviction). */
int fl_dev_time_mul_mat_q(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const void *Yq8, int N,
                          float *dst, size_t dst_row_stride_elems, int impl, int iters, size_t flush_l2_bytes,
                          float *ms_per_launch);
int fl_dev_time_mul_mat_q_rot(int type, const void *W, size_t w_row_stride_bytes, int M, int K, const void *Yq8, int N,
                              float *dst, size_t dst_row_stride_elems, int impl, int iters, size_t flush_l2_bytes,
                              size_t copy_stride_bytes, int n_copies, float *ms_per_launch);

/* ---- the other ops of the LLaMA eval graph, device-resident (SURVEY.md section 8 row f1) ------
 * fl_view is a strided 4-D view in ggml conventions (reference include/ggml.h:279-309): ne[] are
 * element counts, nb[] byte strides.  All tensors f32.  Reference implementations cited in
 * fastllama_b200/csrc/fl_ops_kernels.cu. */
typedef struct fl_view {
    void *data;
    int64_t ne[4];
    int64_t nb[4];
} fl_view;

int fl_dev_rms_norm(const fl_view *src, const fl_view *dst);                 /* eps = 1e-6 (lib/ggml.c:7404) */
int fl_dev_add(const fl_view *a, const fl_view *b, const fl_view *dst);
int fl_dev_mul(const fl_view *a, const fl_view *b, const fl_view *dst);
int fl_dev_repeat(const fl_view *src, const fl_view *dst);
int fl_dev_scale(const fl_view *t, float v);                                /* in place */
int fl_dev_scale_f16(const fl_view *t, float v);                            /* in place, contiguous f16 (fl_dev_add_q_f16 above) */
int fl_dev_silu(const fl_view *src, const fl_view *dst);                    /* fp16-table silu (lib/ggml.c:3207-3215) */
int fl_dev_diag_mask_inf(const fl_view *t, int n_past);                     /* in place */
int fl_dev_soft_max(const fl_view *t);                                      /* in place, fp16-table exp */
int fl_dev_rope(const fl_view *t, int n_past, int n_dims, int mode);        /* in place */
int fl_dev_cpy_f32(const fl_view *src, const fl_view *dst);
int fl_dev_mul_mat_f32(const fl_view *src0, const fl_view *src1, const fl_view *dst);

/* Tensor-parallel prompt ingest: fl_comm_allgather_f32 of every rank's [N][n_local] slice of a row-split result returns
 * [world][N][n_local]; this writes the eval's layout [N][world * n_local] (rank r's slice at columns [r * n_local, +n_local) of
 * every row).  residual (nullable, [N][world * n_local]) is added with one fp32 rounding per element -- the bits of ggml_add --
 * so the gather after wo / w2 needs no separate add.  dst must not overlap `gathered`; it may be `residual`. */
int fl_dev_tp_unshard(const float *gathered, int world, int N, int n_local, const float *residual, float *dst);
/* The same for uneven slices (world 1..8): rank r's [N][count[r]] block sits at gathered + r * N * slice_stride (an all-gather of
 * slices padded to slice_stride floats) and goes to columns [first[r], first[r] + count[r]) of [N][n], n = sum of count[].  first[]
 * and count[] are host arrays of `world` entries; the slices must tile [0, n).  float4 accesses for the ranks whose slice allows
 * them, scalar ones for the others; residual and the overlap rules as above. */
int fl_dev_tp_unshard_v(const float *gathered, int world, int N, int slice_stride, const int *first, const int *count, const float *residual,
                        float *dst);

/* ---- fused decode step (N = 1) ------------------------------------------------------------------
 * fl_dev_mv_fused: up to three weight matrices that share one input, one launch.  The prologue builds
 * the q8_0 activations from f32 inside the kernel (replacing rms_norm / mul / silu / quantize_row_q8_0
 * launches, reference lib/ggml.c:7378-7434, :3207-3215, :1299-1441); the epilogue replaces the
 * ggml_add after wo / w2 or the rope + KV-cache copies after wq|wk|wv (reference lib/llama.cpp:328-343).
 * All pointers are device pointers.  n_past is read on the device (CUDA-graph replay). */
enum { FL_PRO_PLAIN = 0, FL_PRO_RMSNORM = 1, FL_PRO_SILUMUL = 2 };
enum { FL_EPI_STORE = 0, FL_EPI_RESADD = 1, FL_EPI_QKV = 2 };
typedef struct fl_mv_args {
    int type, K, nseg;
    const void *seg_w[3];        /* weight matrices: seg_rows[i] rows of K/32 blocks, contiguous rows */
    int seg_rows[3];
    float *seg_dst[3];           /* f32 outputs (EPI_QKV: only seg_dst[0] = q buffer is used) */
    int pro;
    const float *x;              /* PRO_PLAIN / PRO_RMSNORM input; PRO_SILUMUL: the silu argument */
    const float *gamma;          /* PRO_RMSNORM: norm weight */
    const float *b;              /* PRO_SILUMUL: the multiplier */
    float *normed_out;           /* PRO_RMSNORM: optional copy of gamma * rms_norm(x) (the "embeddings") */
    const float *xadd;           /* optional: the prologue input is x + xadd ... */
    float *sum_out;              /* ... and x + xadd is also written here (by CTA 0) */
    size_t row_stride_bytes;     /* 0 = dense rows of K/32 blocks; else the (16-B multiple) stride of packed K-slices */
    const uint16_t *silu_tab;    /* filled in by the library */
    int epi;
    const float *res;            /* EPI_RESADD */
    const int *n_past;           /* EPI_QKV ... */
    int n_ctx, n_embd, head_dim;
    const void *rope_cs;         /* filled in by the library (cos/sin table) */
    float *kcache, *vcache;      /* this layer's K [pos][n_embd] and V [n_embd][n_ctx] cache */
    /* Dataflow vectors of the token kernel (fl_token_plan_*, never fl_dev_mv_fused).  A vector in "LL" form holds one 8-byte word
     * {value, epoch} per element, so a consumer sees the arrival of every element by itself and NO grid barrier (local or cross-GPU)
     * separates the producing step from the consuming one; the library keeps the running epoch (epoch = launches so far * exchanges
     * per launch + seq + 1) next to the buffers.
     *   x_ll:   x is an LL vector written by an earlier step of this token under sequence number x_seq: the prologue polls until every
     *           element carries that epoch, and the grid barrier in front of the step is dropped.
     *   out_ll: seg_dst[0] is an LL vector (element r at byte 8r): output row r is stored as {value, epoch(out_seq)}.  With
     *           n_dst_peer > 0 the same word also goes to dst_peer[0..n_dst_peer) -- the same vector in every other rank's buffer, over
     *           NVLink (fl_comm_shared_alloc): a ROW-split step of a tensor-parallel model passes pointers that are pre-offset by its
     *           first row, so every rank ends up with the complete gathered vector, bit-identical to the one-GPU run.
     *   res_ll: EPI_RESADD reads the residual from an LL vector (element r at res[2r]) that an earlier step has polled completely.
     * SwiGLU pairs (w1|w3, see fl_token_kernel.cu) store silu(a)*b the same way when out_ll is set. */
    float *dst_peer[7];
    int n_dst_peer;
    int x_ll, x_seq, out_ll, out_seq, res_ll;
    int swiglu;                  /* nseg == 2 (w1|w3 of the FFN): store silu(seg 0 . x) * (seg 1 . x) to seg_dst[0]; seg_dst[1] is not written.
                                    (Plans without this flag get the same fusion when the next step is the matching PRO_SILUMUL.) */
} fl_mv_args;
int fl_dev_mv_fused_supported(int type, int K, int mtot);
int fl_dev_mv_fused(const fl_mv_args *args);
/* attention of one new token over the cached positions 0..n_past (reference lib/llama.cpp:346-398, N = 1) */
int fl_dev_attn_decode(const float *q, const float *kcache, const float *vcache, float *out, const int *n_past, int k_row_stride,
                       int n_head, int head_dim, int n_ctx, float scale);   /* k_row_stride = n_embd of the model (floats per cached position) */
int fl_dev_rope_table(int n_dims, int n_pos);    /* make sure the cos/sin table covers n_pos positions */

/* ---- the whole decode step as one persistent kernel ---------------------------------------------
 * A token plan is a list of steps, each either an fl_dev_mv_fused call (kind 0) or an
 * fl_dev_attn_decode call (kind 1) with exactly the arguments above; fl_token_plan_launch runs them in
 * order inside ONE cooperative launch of one CTA per SM, with the weight stream prefetched across steps.  Steps are separated by grid
 * barriers unless the consumer's input is a dataflow ("LL") vector (x_ll), in which case the elements themselves signal arrival. */
typedef struct fl_token_step {
    int kind;                    /* 0 = matvec (mv), 1 = attention (the fields below) */
    fl_mv_args mv;
    const float *q, *kcache, *vcache;
    float *out;
    const int *n_past;
    int k_row_stride, n_head, head_dim, n_ctx;
    float scale;
    /* attention output as an LL vector (see fl_mv_args): element h * head_dim + d of out / out_peer[] */
    int out_ll, out_seq, n_out_peer;
    float *out_peer[7];
} fl_token_step;
int fl_token_plan_create(const fl_token_step *steps, int n_steps, void **plan_out);
/* the same for steps that use LL vectors: epoch_counter is a zero-initialised device word that lives (and is freed) WITH the LL vectors and
 * is shared by every plan that uses them -- the kernel advances it by the number of exchanges per launch */
int fl_token_plan_create_ll(const fl_token_step *steps, int n_steps, unsigned *epoch_counter, void **plan_out);
int fl_token_plan_launch(void *plan);
int fl_token_plan_destroy(void *plan);
/* nonzero after a launch whose in-kernel barriers timed out (a peer never arrived); the results are then invalid */
int fl_token_plan_error(void *plan);
/* tooling: with FASTLLAMA_B200_TOKEN_PROF set at create time, the last launch's per-step, per-CTA timestamps
 * [n_steps][n_ctas][4] in ns: step entered, grid barrier passed, activations quantised, tiles consumed */
int fl_token_plan_profile(void *plan, unsigned long long *out, size_t max_words, int *n_ctas);
/* tooling: per step, CTA and consumer warp [n_steps][n_ctas][16][8] SM-clock cycle counts of the last launch's tile loops:
 * activation fetch, waiting for weight tiles, dot products, reduction + epilogue, rounds, total, tiles of the CTA, 0 */
int fl_token_plan_profile2(void *plan, unsigned *out, size_t max_words);

/* ---- tensor parallelism (SURVEY.md 8e): one process per GPU, NCCL (dlopen'ed libnccl.so.2) on the
 * library stream; collectives are captured into the decode CUDA graph.  fl_comm_unique_id is called on
 * rank 0 and its 128 bytes are distributed by the launcher (bench.py uses torch.distributed). */
int fl_comm_unique_id(void *out128);
int fl_comm_init(int rank, int world, const void *id128);
int fl_comm_rank(void);
int fl_comm_world(void);
int fl_comm_allreduce_f32(float *buf_dev, size_t n);                                   /* in place, sum */
int fl_comm_allgather_f32(const float *send_dev, float *recv_dev, size_t n_per_rank);
/* Peer-visible scratch for collectives fused into the token kernel: every rank allocates `bytes` (zeroed) of device
 * memory, the CUDA IPC handles travel through the NCCL communicator, and each rank maps the others' buffers over
 * NVLink.  peers_out[r] = pointer, valid on THIS rank, to rank r's buffer (r = own rank: the local allocation).
 * The caller lays the buffer out (libggml_b200: 4096 bytes of counters, then the dataflow vectors of the decode step).  Collective
 * call; returns nonzero when peer mapping is unavailable (tensor-parallel decode then refuses to run: its gathers need peer memory). */
int fl_comm_shared_alloc(size_t bytes, void **peers_out);
/* copy blocks [blk0, blk0 + nblk) of every row of a quantised matrix into a packed matrix whose row
 * stride is dst_row_stride bytes (a column slice; not used by the decode plan any more: every matrix is row-split) */
int fl_dev_pack_cols(int type, const void *W, size_t w_row_stride_bytes, int M, int blk0, int nblk, void *dst, size_t dst_row_stride);

/* CUDA-graph capture of everything issued on the library stream between begin and end */
int fl_graph_begin_capture(void);
int fl_graph_end_capture(void **graph_exec_out);
int fl_graph_launch(void *graph_exec);
int fl_graph_destroy(void *graph_exec);

/* Tooling: counter-based N(0, std^2) fill (element i depends on (seed, i) only) used to create
 * synthetic model files on the device; not part of the hot path. */
int fl_dev_fill_normal(float *p_dev, size_t n, uint64_t seed, float std);

/* CUDA events on the library stream (device-side timing for the graph executor and bench.py) */
void *fl_event_create(void);
int fl_event_destroy(void *ev);
int fl_event_record(void *ev);
int fl_event_sync(void *ev);
int fl_event_elapsed_ms(void *ev_start, void *ev_stop, float *ms);

/* number of kernels this library has launched since fl_init (bench.py "gpu_launches") */
uint64_t fl_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FL_CUDA_H */
