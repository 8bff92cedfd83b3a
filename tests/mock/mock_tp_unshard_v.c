/*
 * mock_tp_unshard_v.c -- TEST-ONLY CPU stand-in for fl_dev_tp_unshard_v (include/fl_cuda.h).
 *
 * tests/test_tp_uneven.py links it together with mock_fl_cuda.c, mock_tp_unshard.c and the oracle into one CPU libfl_cuda.so, so that
 * the tensor-parallel plans of libggml_b200 run at uneven world sizes over gloo without a GPU.  Rank r's [N][count[r]] block at
 * g + r * N * stride -> columns [first[r], first[r] + count[r]) of [N][sum of count], + residual with one fp32 rounding per element.
 */
#include <stddef.h>

int fl_dev_tp_unshard_v(const float *g, int world, int N, int stride, const int *first, const int *count, const float *res, float *d) {
    if (!g || !d || !first || !count || world < 1 || world > 8 || N < 0 || stride < 0) return -1;
    int n = 0;
    for (int r = 0; r < world; r++) {
        if (count[r] < 0 || count[r] > stride || first[r] < 0) return -1;
        n += count[r];
    }
    for (int r = 0; r < world; r++)
        for (int c = 0; c < N; c++)
            for (int j = 0; j < count[r]; j++) {
                const size_t o = (size_t)c * n + first[r] + j;
                const float v = g[((size_t)r * N) * stride + (size_t)c * count[r] + j];
                d[o] = res ? v + res[o] : v;
            }
    return 0;
}
