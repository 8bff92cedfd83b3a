/*
 * fl_ggml.h -- drop-in boundary B1: the slice of the reference's ggml C API that the LLaMA eval
 * path is built on, re-implemented by libggml_b200 on top of the CUDA layer (fl_cuda.h).
 *
 * This header is written for THIS repository's own C/C++ code and tests.  The reference's
 * lib/llama.cpp and lib/bridge.cpp are compiled UNCHANGED against their own include/ggml.h; what
 * makes the swap possible is that libggml_b200 exports the same symbols with the same ABI:
 *   - struct layouts  : reference include/ggml.h:267-342 (ggml_object 32 B, ggml_tensor 176 B,
 *                       ggml_cgraph 98360 B, ggml_scratch, ggml_init_params) -- checked by
 *                       static_asserts below and by tests/test_ggml_abi.py against the reference;
 *   - enum numbering  : ggml_type 0..9 (a model-file contract, include/ggml.h:201-214) and ggml_op
 *                       (include/ggml.h:217-263);
 *   - function set    : the 41 ggml_* symbols the reference's upper layers import (listed in
 *                       INTEGRATION.md, obtained with `nm -u`) plus the helpers declared here;
 *   - semantics       : tensors are bump-allocated inside the caller's buffer with the reference's
 *                       exact space accounting (lib/ggml.c:3809-3928); ggml_graph_compute is
 *                       synchronous from the caller's view (results the caller reads are in host
 *                       memory on return, SURVEY.md 8b).
 *
 * What differs, by design: ggml_graph_compute runs the graph on the GPU (weights, KV cache and
 * activations live in device mirrors of the host arenas); cgraph->n_threads is ignored; ops outside
 * the LLaMA eval set abort with a message instead of silently running on the CPU.
 */
#ifndef FL_GGML_H
#define FL_GGML_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GGML_MAX_DIMS 4
#define GGML_MAX_NODES 4096
#define GGML_MAX_OPT 4
#define GGML_MAX_CONTEXTS 64
#define GGML_DEFAULT_N_THREADS 4

typedef uint16_t ggml_fp16_t;

enum ggml_type {
    GGML_TYPE_F32 = 0, GGML_TYPE_F16 = 1, GGML_TYPE_Q4_0 = 2, GGML_TYPE_Q4_1 = 3, GGML_TYPE_Q4_2 = 4,
    GGML_TYPE_Q4_3 = 5, GGML_TYPE_Q8_0 = 6, GGML_TYPE_I8 = 7, GGML_TYPE_I16 = 8, GGML_TYPE_I32 = 9,
    GGML_TYPE_COUNT = 10
};

/* same order as the reference so the integer values agree */
enum ggml_op {
    GGML_OP_NONE = 0, GGML_OP_DUP, GGML_OP_ADD, GGML_OP_SUB, GGML_OP_MUL, GGML_OP_DIV, GGML_OP_SQR,
    GGML_OP_SQRT, GGML_OP_SUM, GGML_OP_MEAN, GGML_OP_REPEAT, GGML_OP_ABS, GGML_OP_SGN, GGML_OP_NEG,
    GGML_OP_STEP, GGML_OP_RELU, GGML_OP_GELU, GGML_OP_SILU, GGML_OP_NORM, GGML_OP_RMS_NORM,
    GGML_OP_MUL_MAT, GGML_OP_SCALE, GGML_OP_CPY, GGML_OP_CONT, GGML_OP_RESHAPE, GGML_OP_VIEW,
    GGML_OP_PERMUTE, GGML_OP_TRANSPOSE, GGML_OP_GET_ROWS, GGML_OP_DIAG_MASK_INF, GGML_OP_SOFT_MAX,
    GGML_OP_ROPE, GGML_OP_CONV_1D_1S, GGML_OP_CONV_1D_2S, GGML_OP_FLASH_ATTN, GGML_OP_FLASH_FF,
    GGML_OP_MAP_UNARY, GGML_OP_MAP_BINARY, GGML_OP_COUNT
};

struct ggml_context;

struct ggml_object {            /* arena bookkeeping record that precedes every tensor */
    size_t offs, size;
    struct ggml_object *next;
    char padding[8];
};

struct ggml_tensor {
    enum ggml_type type;
    int n_dims;
    int64_t ne[GGML_MAX_DIMS];  /* element counts, fastest first */
    size_t nb[GGML_MAX_DIMS];   /* byte strides */
    enum ggml_op op;
    bool is_param;
    struct ggml_tensor *grad, *src0, *src1;
    struct ggml_tensor *opt[GGML_MAX_OPT];
    int n_tasks;
    int perf_runs;
    int64_t perf_cycles, perf_time_us;
    void *data;                 /* HOST address; the backend maps it to its device mirror */
    char padding[8];
};

struct ggml_cgraph {
    int n_nodes, n_leafs, n_threads;
    size_t work_size;
    struct ggml_tensor *work;
    struct ggml_tensor *nodes[GGML_MAX_NODES];
    struct ggml_tensor *grads[GGML_MAX_NODES];
    struct ggml_tensor *leafs[GGML_MAX_NODES];
    int perf_runs;
    int64_t perf_cycles, perf_time_us;
};

struct ggml_scratch { size_t offs, size; void *data; };
struct ggml_init_params { size_t mem_size; void *mem_buffer; bool no_alloc; };

#ifdef __cplusplus
static_assert(sizeof(struct ggml_object) == 32, "ggml_object ABI");
static_assert(sizeof(struct ggml_tensor) == 176, "ggml_tensor ABI");
static_assert(sizeof(struct ggml_cgraph) == 98360, "ggml_cgraph ABI");
static_assert(sizeof(struct ggml_init_params) == 24, "ggml_init_params ABI");
#endif

/* ---- misc ------------------------------------------------------------------------------- */
void ggml_time_init(void);
int64_t ggml_time_ms(void);
int64_t ggml_time_us(void);
float ggml_fp16_to_fp32(ggml_fp16_t x);
ggml_fp16_t ggml_fp32_to_fp16(float x);
int ggml_cpu_has_blas(void);     /* 0: keeps Model::eval on the n_threads path (lib/llama.cpp:299) */
int ggml_cpu_has_cublas(void);   /* 0: the reference's dead cuBLAS branch is not what this is */

int64_t ggml_nelements(const struct ggml_tensor *t);
size_t ggml_nbytes(const struct ggml_tensor *t);
int ggml_blck_size(enum ggml_type type);
size_t ggml_type_size(enum ggml_type type);
float ggml_type_sizef(enum ggml_type type);
const char *ggml_type_name(enum ggml_type type);
size_t ggml_element_size(const struct ggml_tensor *t);
bool ggml_is_quantized(enum ggml_type type);

/* ---- contexts and tensors (reference lib/ggml.c:3666-4075) ----------------------------------- */
struct ggml_context *ggml_init(struct ggml_init_params params);
void ggml_free(struct ggml_context *ctx);
size_t ggml_used_mem(const struct ggml_context *ctx);
size_t ggml_set_scratch(struct ggml_context *ctx, struct ggml_scratch scratch);

struct ggml_tensor *ggml_new_tensor(struct ggml_context *ctx, enum ggml_type type, int n_dims, const int64_t *ne);
struct ggml_tensor *ggml_new_tensor_1d(struct ggml_context *ctx, enum ggml_type type, int64_t ne0);
struct ggml_tensor *ggml_new_tensor_2d(struct ggml_context *ctx, enum ggml_type type, int64_t ne0, int64_t ne1);
struct ggml_tensor *ggml_new_tensor_3d(struct ggml_context *ctx, enum ggml_type type, int64_t ne0, int64_t ne1, int64_t ne2);
struct ggml_tensor *ggml_new_tensor_4d(struct ggml_context *ctx, enum ggml_type type, int64_t ne0, int64_t ne1, int64_t ne2, int64_t ne3);
struct ggml_tensor *ggml_new_i32(struct ggml_context *ctx, int32_t value);
struct ggml_tensor *ggml_new_f32(struct ggml_context *ctx, float value);
struct ggml_tensor *ggml_dup_tensor(struct ggml_context *ctx, const struct ggml_tensor *src);
struct ggml_tensor *ggml_view_tensor(struct ggml_context *ctx, const struct ggml_tensor *src);
struct ggml_tensor *ggml_set_zero(struct ggml_tensor *t);
struct ggml_tensor *ggml_set_i32(struct ggml_tensor *t, int32_t value);
struct ggml_tensor *ggml_set_f32(struct ggml_tensor *t, float value);
void *ggml_get_data(const struct ggml_tensor *t);
float *ggml_get_data_f32(const struct ggml_tensor *t);

/* ---- graph builders (reference lib/ggml.c:4266-5420); host-only, no device work ---------------- */
struct ggml_tensor *ggml_dup(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_add(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_add_inplace(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_mul(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_repeat(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_silu(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_rms_norm(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_mul_mat(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_scale(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_cpy(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_cont(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_reshape(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_reshape_2d(struct ggml_context *ctx, struct ggml_tensor *a, int64_t ne0, int64_t ne1);
struct ggml_tensor *ggml_reshape_3d(struct ggml_context *ctx, struct ggml_tensor *a, int64_t ne0, int64_t ne1, int64_t ne2);
struct ggml_tensor *ggml_view_1d(struct ggml_context *ctx, struct ggml_tensor *a, int64_t ne0, size_t offset);
struct ggml_tensor *ggml_view_2d(struct ggml_context *ctx, struct ggml_tensor *a, int64_t ne0, int64_t ne1, size_t nb1, size_t offset);
struct ggml_tensor *ggml_view_3d(struct ggml_context *ctx, struct ggml_tensor *a, int64_t ne0, int64_t ne1, int64_t ne2, size_t nb1, size_t nb2, size_t offset);
struct ggml_tensor *ggml_permute(struct ggml_context *ctx, struct ggml_tensor *a, int axis0, int axis1, int axis2, int axis3);
struct ggml_tensor *ggml_transpose(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_get_rows(struct ggml_context *ctx, struct ggml_tensor *a, struct ggml_tensor *b);
struct ggml_tensor *ggml_diag_mask_inf(struct ggml_context *ctx, struct ggml_tensor *a, int n_past);
struct ggml_tensor *ggml_soft_max(struct ggml_context *ctx, struct ggml_tensor *a);
struct ggml_tensor *ggml_rope(struct ggml_context *ctx, struct ggml_tensor *a, int n_past, int n_dims, int mode);

void ggml_build_forward_expand(struct ggml_cgraph *cgraph, struct ggml_tensor *tensor);
struct ggml_cgraph ggml_build_forward(struct ggml_tensor *tensor);

/* Runs the graph on the GPU (replaces ggml_graph_compute + the pthread pool, reference
 * lib/ggml.c:10811-11253, and the per-op ggml_compute_forward_* switch :10117-10285).  Aborts with a
 * message (like GGML_ASSERT) on an op/type outside the LLaMA eval set or on any CUDA error. */
void ggml_graph_compute(struct ggml_context *ctx, struct ggml_cgraph *cgraph);

/* ---- quantisation entry points ---------------------------------------------------------------- */
size_t ggml_quantize_q4_0(const float *src, void *dst, int n, int k, int64_t *hist);
size_t ggml_quantize_q4_1(const float *src, void *dst, int n, int k, int64_t *hist);
size_t ggml_quantize_chunk(enum ggml_type type, const float *src, void *dst, int start, int n, int64_t *hist);

typedef void (*dequantize_row_q_t)(const void *x, float *y, int k);
typedef void (*quantize_row_q_t)(const float *x, void *y, int k);
typedef void (*vec_dot_q_t)(const int n, float *s, const void *x, const void *y);
typedef struct {
    dequantize_row_q_t dequantize_row_q;
    quantize_row_q_t quantize_row_q;
    quantize_row_q_t quantize_row_q_reference;
    quantize_row_q_t quantize_row_q_dot;
    vec_dot_q_t vec_dot_q;
} quantize_fns_t;
/* the reference's test hook (include/ggml.h:841-862); here every pointer runs the CUDA kernels */
quantize_fns_t ggml_internal_get_quantize_fn(size_t i);

/* ---- backend controls (ours; not part of the reference surface) -------------------------------- */
/* Host code changed bytes inside [ptr, ptr+size) of a persistent arena (weights after a LoRA merge,
 * KV cache after load_state): re-upload that range before the next graph. */
void ggml_b200_invalidate(const void *ptr, size_t size);
/* Copy a device-resident range back to its host arena (KV cache before save_state). */
void ggml_b200_sync_to_host(const void *ptr, size_t size);
/* Free every device resource of the backend: all contexts' mirrors, decode states, shards and workspaces (all models unloaded). */
void ggml_b200_release_all(void);
/* Free the device resources of everything whose host memory is gone: mirrors of freed arenas and of unmapped or remapped file ranges,
 * decode states of freed contexts, tensor-parallel shards of freed weights, and the shared workspaces once no context is left.  Live
 * contexts keep everything, their device-written KV caches included.  fastllama_b200.Model.close() calls it after llama_free_context;
 * after the last context it leaves the device as ggml_b200_release_all does. */
void ggml_b200_release_unused(void);
/* Contexts of this process:
 *   live_states:       decode states (one per context that has run an eval on the fused plans; released with the context);
 *   plan_builds:       token-kernel programs built so far (a plan is built once per context and shape, not per switch);
 *   graph_captures:    decode steps captured into a CUDA graph so far;
 *   external_copies:   device copies of mmap'ed weight ranges, keyed by (file, offset): mappings of one file share them;
 *   external_mappings: live mapped ranges using those copies (> external_copies when contexts share a file);
 *   external_bytes:    bytes of those copies. */
struct ggml_b200_contexts { uint64_t live_states, plan_builds, graph_captures, external_copies, external_mappings, external_bytes; };
void ggml_b200_get_contexts(struct ggml_b200_contexts *out);
/* Counters for bench.py: evals run, device microseconds of the last eval (CUDA events), kernels launched */
struct ggml_b200_stats { uint64_t n_evals; double last_eval_device_us; double total_device_us; uint64_t launches; uint64_t graph_replays; };
void ggml_b200_get_stats(struct ggml_b200_stats *out);
/* Profile mode (bench.py roofline leg): every quantised mul_mat launch is bracketed by CUDA events on
 * the launching stream and accumulated per (type, M, K, N).  algo_bytes = M*(K/32)*block + (K/32)*40*N
 * + 4*M*N per launch (SURVEY.md 8d).  Turning it on resets the table. */
struct ggml_b200_kernel_stat { int type, M, K, N; uint64_t launches; double total_ms; double algo_bytes_per_launch; };
void ggml_b200_set_profile(int on);
int ggml_b200_get_kernel_stats(struct ggml_b200_kernel_stat *out, int max_entries);
/* how the last single-token eval ran: 0 = node-by-node executor, 1 = fused plan, one kernel per matrix group,
 * 2 = fused plan as one persistent kernel per token (fl_token_kernel.cu) */
int ggml_b200_decode_mode(void);
/* host-side time of the fused decode path in microseconds, summed over decode steps: [0] steps, [1] graph match, [2] match + scalars +
 * launch issue, [3] waiting for the device + result copies, [4] time spent in the caller between two decode steps */
void ggml_b200_get_host_profile(double out[8], int reset);
/* how the last multi-token eval ran: 0 = node-by-node executor (every rank replicated under tensor parallelism), 1 = tensor-parallel
 * prompt plan (row-split matrices on this rank's weight shards, activations all-gathered; FASTLLAMA_B200_TP_INGEST=replicated forces 0) */
int ggml_b200_prompt_mode(void);
/* Device memory of this process:
 *   weight_mirror_bytes: device mirrors of arenas / mmap ranges that the executor has read model weights from (0 on a
 *                        tensor-parallel rank that has only run decode steps and prompt-plan evals: no rank copies the model);
 *   shard_bytes:         tensor-parallel weight shards (this rank's rows of every matrix, norm weights, embedding table);
 *   mirror_bytes:        all device mirrors (weights, KV cache, compute and scratch arenas);
 *   kv_gathers:          all-gathers of a head-sharded KV cache run so far (save_state, or an eval that needs every head). */
struct ggml_b200_memory { uint64_t weight_mirror_bytes, shard_bytes, mirror_bytes, kv_gathers; };
void ggml_b200_get_memory(struct ggml_b200_memory *out);

#ifdef __cplusplus
}
#endif
#endif /* FL_GGML_H */
