/*
 * mock_quantize_file_lora.c -- TEST-ONLY CPU stand-in for fl_dev_quantize_q4_file_lora (include/fl_cuda.h).
 *
 * Each row is merged with its delta the way the reference's ggml_add_inplace merges it into an unquantised model
 * (f32 file: w + d; f16 file: fp16_rn(w + fp32(d)) with F16C's _cvtss_sh, round to nearest even), then quantised
 * as f32 by the stand-in's fl_dev_quantize_q4_file.  Without a delta it is that function (source type 3, f16 data
 * of an f32 file, as 1).
 *
 * tests/test_quantize_lora.py links it with mock_quantize_file_f16round.c, mock_fl_cuda.c and the oracle into one
 * CPU libfl_cuda.so, with -Bsymbolic so that the call to fl_dev_quantize_q4_file below binds to that library's own
 * definition even when the real libfl_cuda.so is already loaded into the process with RTLD_GLOBAL.
 */
#include <immintrin.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

int fl_dev_quantize_q4_file(int type, int src_type, const void *x, void *y, int k, int nrows, unsigned long long *hist);

int fl_dev_quantize_q4_file_lora(int type, int src_type, const void *x, int delta_type, const void *delta, void *y, int k, int nrows,
                                 unsigned long long *hist) {
    if ((type != 2 && type != 3) || src_type < 0 || src_type > 3 || delta_type < -1 || delta_type > 1 || (delta_type == -1) != (delta == NULL) ||
        (delta_type == 1 && (src_type == 0 || src_type == 3)) || k <= 0 || k % 32) {
        fprintf(stderr, "fl_dev_quantize_q4_file_lora: bad arguments (type %d, src_type %d, delta_type %d, k %d)\n", type, src_type, delta_type, k);
        return -1;
    }
    if (delta_type == -1) return fl_dev_quantize_q4_file(type, src_type == 3 ? 1 : src_type, x, y, k, nrows, hist);
    const size_t row_bytes = (size_t)(k / 32) * (type == 2 ? 20 : 24);
    float *row = malloc((size_t)k * sizeof(float));
    if (!row) return -1;
    int rc = 0;
    for (int r = 0; r < nrows && rc == 0; r++) {
        for (int i = 0; i < k; i++) {
            const size_t e = (size_t)r * k + i;
            float w;
            if (src_type == 1 || src_type == 3) w = _cvtsh_ss(((const uint16_t *)x)[e]);
            else if (src_type == 2) w = (float)(_Float16)((const float *)x)[e];
            else w = ((const float *)x)[e];
            const float d = delta_type == 1 ? _cvtsh_ss(((const uint16_t *)delta)[e]) : ((const float *)delta)[e];
            float s = w + d;
            if (src_type == 1 || src_type == 2) s = _cvtsh_ss(_cvtss_sh(s, 0));
            row[i] = s;
        }
        rc = fl_dev_quantize_q4_file(type, 0, row, (uint8_t *)y + (size_t)r * row_bytes, k, 1, hist);
    }
    free(row);
    return rc;
}
