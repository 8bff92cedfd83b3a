/*
 * mock_quantize_file_f16round.c -- TEST-ONLY CPU stand-in for fl_dev_quantize_q4_file (include/fl_cuda.h)
 * with every source type: 0 (f32) and 1 (f16) are mock_quantize_file.c's, included here under another
 * name; 2 (f32 rounded to f16 and widened back) rounds each row with a (_Float16) cast, which gcc on
 * x86-64 rounds to nearest even like numpy's astype(float16), and quantises it as f32.
 *
 * tests/test_quantize_checkpoint.py links it, in place of mock_quantize_file.c, with mock_fl_cuda.c and
 * the oracle into one CPU libfl_cuda.so.
 */
#define fl_dev_quantize_q4_file mock_quantize_q4_file_f32_f16
#include "mock_quantize_file.c"
#undef fl_dev_quantize_q4_file

int fl_dev_quantize_q4_file(int type, int src_type, const void *x, void *y, int k, int nrows, unsigned long long *hist) {
    if (src_type != 2 || (type != 2 && type != 3) || k <= 0 || k % 32)
        return mock_quantize_q4_file_f32_f16(type, src_type, x, y, k, nrows, hist);
    const size_t row_bytes = (size_t)(k / 32) * (type == 2 ? 20 : 24);
    float *row = malloc((size_t)k * sizeof(float));
    if (!row) return -1;
    int rc = 0;
    for (int r = 0; r < nrows && rc == 0; r++) {
        for (int i = 0; i < k; i++) row[i] = (float)(_Float16)((const float *)x)[(size_t)r * k + i];
        rc = mock_quantize_q4_file_f32_f16(type, 0, row, (uint8_t *)y + (size_t)r * row_bytes, k, 1, hist);
    }
    free(row);
    return rc;
}
