/*
 * lora_f16_oracle.c -- TEST INFRASTRUCTURE ONLY.  C restatement of the two ops behind a cached f16 LoRA adapter
 * (scripts/convert-lora-to-ggml.py --dtype fp16) in the reference's x86 build (AVX2 / FMA / F16C), on top of the row
 * functions of oracle/q4_oracle.c, with which it is compiled and linked.  Pinned by tests/golden/lora_f16_ops.npz.
 */
#include <immintrin.h>      /* _cvtsh_ss / _cvtss_sh: the F16C conversions of GGML_FP16_TO_FP32 / GGML_FP32_TO_FP16 */
#include <stdint.h>
#include <stdlib.h>

int orc_block_bytes(int ggml_type);
void orc_dequantize_row_q4_0(const void *vx, float *y, int k);
void orc_dequantize_row_q4_1(const void *vx, float *y, int k);
void orc_quantize_row_q4_0_simd(const float *x, void *vy, int k);
void orc_quantize_row_q4_1_simd(const float *x, void *vy, int k);

/* ggml_compute_forward_add_q_f16 (lib/ggml.c:12372-12483): dst row = quantize_row_q(dequantize_row_q(src0 row) + fp32(src1 row)),
 * the SIMD quantiser, each f16 element widened exactly before the one fp32 add.  Rows are dense. */
int orc_add_q_f16(int ggml_type, int rows, int k, const void *src0, const uint16_t *src1, void *dst) {
    const int bb = orc_block_bytes(ggml_type);
    if (bb < 0 || (ggml_type != 2 && ggml_type != 3) || k % 32) return -1;
    float *w = (float *)malloc(sizeof(float) * (size_t)k);
    if (!w) return -1;
    for (int r = 0; r < rows; r++) {
        const uint8_t *s0 = (const uint8_t *)src0 + (size_t)r * (k / 32) * bb;
        uint8_t *d = (uint8_t *)dst + (size_t)r * (k / 32) * bb;
        if (ggml_type == 2) orc_dequantize_row_q4_0(s0, w, k); else orc_dequantize_row_q4_1(s0, w, k);
        for (int i = 0; i < k; i++) w[i] += _cvtsh_ss(src1[(size_t)r * k + i]);
        if (ggml_type == 2) orc_quantize_row_q4_0_simd(w, d, k); else orc_quantize_row_q4_1_simd(w, d, k);
    }
    free(w);
    return 0;
}

/* ggml_compute_forward_scale_f16 (lib/ggml.c:12485-12524), in place on n contiguous f16 values: x = fp16(fp32(x) * v), round to
 * nearest even (_cvtss_sh(., 0)) */
void orc_scale_f16(uint16_t *x, long n, float v) {
    for (long i = 0; i < n; i++) x[i] = _cvtss_sh(_cvtsh_ss(x[i]) * v, 0);
}
