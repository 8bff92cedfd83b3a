/*
 * mock_quantize_file.c -- TEST-ONLY CPU stand-in for fl_dev_quantize_q4_file (include/fl_cuda.h).
 *
 * tests/test_quantize_model.py links it together with mock_fl_cuda.c and the oracle into one CPU
 * libfl_cuda.so, so that fastllama_b200/quantize.py runs end to end without a GPU.  The arithmetic is
 * the oracle's quantize_row_q4_{0,1}_reference restatement; f16 inputs are widened exactly (F16C).
 */
#include <immintrin.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

void orc_quantize_row_q4_0(const float *x, void *vy, int k);
void orc_quantize_row_q4_1(const float *x, void *vy, int k);

int fl_dev_quantize_q4_file(int type, int src_type, const void *x, void *y, int k, int nrows, unsigned long long *hist) {
    if ((type != 2 && type != 3) || (src_type != 0 && src_type != 1) || k <= 0 || k % 32) {
        fprintf(stderr, "fl_dev_quantize_q4_file: bad arguments (type %d, src_type %d, k %d)\n", type, src_type, k);
        return -1;
    }
    const int bb = type == 2 ? 20 : 24, qoff = type == 2 ? 4 : 8;
    float *row = malloc((size_t)k * sizeof(float));
    if (!row) return -1;
    for (int r = 0; r < nrows; r++) {
        if (src_type == 1)
            for (int i = 0; i < k; i++) row[i] = _cvtsh_ss(((const uint16_t *)x)[(size_t)r * k + i]);
        else
            memcpy(row, (const float *)x + (size_t)r * k, (size_t)k * sizeof(float));
        uint8_t *yr = (uint8_t *)y + (size_t)r * (k / 32) * bb;
        if (type == 2) orc_quantize_row_q4_0(row, yr, k); else orc_quantize_row_q4_1(row, yr, k);
        if (hist)
            for (int b = 0; b < k / 32; b++)
                for (int j = 0; j < 16; j++) { hist[yr[b * bb + qoff + j] & 0xF]++; hist[yr[b * bb + qoff + j] >> 4]++; }
    }
    free(row);
    return 0;
}
