/*
 * mock_lora_f16.c -- TEST-ONLY CPU stand-ins for fl_dev_add_q_f16 and fl_dev_scale_f16 (include/fl_cuda.h), built on the oracle's
 * restatement (oracle/lora_f16_oracle.c).  tests/lora_mock.py links it together with mock_fl_cuda.c and the oracle into one CPU
 * libfl_cuda.so, so that cached f16 LoRA adapters run through libggml_b200 without a GPU.
 */
#include <stddef.h>
#include <stdint.h>

#include "fl_cuda.h"

int orc_add_q_f16(int ggml_type, int rows, int k, const void *src0, const uint16_t *src1, void *dst);
void orc_scale_f16(uint16_t *x, long n, float v);

int fl_dev_add_q_f16(int type, const void *W, size_t wrs, int M, int K, const uint16_t *X, size_t xrs, void *dst, size_t drs) {
    for (int r = 0; r < M; r++)
        if (orc_add_q_f16(type, 1, K, (const char *)W + (size_t)r * wrs, X + (size_t)r * xrs, (char *)dst + (size_t)r * drs)) return -1;
    return 0;
}

int fl_dev_scale_f16(const fl_view *t, float v) {
    int64_t nb = 2, n = 1;
    for (int i = 0; i < 4; i++) {
        if (t->nb[i] != nb) return -1;           /* contiguous f16 only, as ggml_compute_forward_scale_f16 asserts */
        nb *= t->ne[i];
        n *= t->ne[i];
    }
    orc_scale_f16((uint16_t *)t->data, (long)n, v);
    return 0;
}
