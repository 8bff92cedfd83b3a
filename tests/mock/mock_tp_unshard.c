/*
 * mock_tp_unshard.c -- TEST-ONLY CPU stand-in for fl_dev_tp_unshard (include/fl_cuda.h).
 *
 * tests/test_tp_ingest.py links it together with mock_fl_cuda.c and the oracle into one CPU libfl_cuda.so, so that the
 * tensor-parallel prompt plan of libggml_b200 runs over gloo without a GPU.  [world][N][n_local] -> [N][world * n_local],
 * + residual with one fp32 rounding per element.
 */
#include <stddef.h>

int fl_dev_tp_unshard(const float *g, int world, int N, int nl, const float *res, float *d) {
    if (!g || !d || world < 1 || N < 0 || nl < 0) return -1;
    for (int n = 0; n < N; n++)
        for (int r = 0; r < world; r++)
            for (int j = 0; j < nl; j++) {
                const size_t o = ((size_t)n * world + r) * nl + j;
                const float v = g[((size_t)r * N + n) * nl + j];
                d[o] = res ? v + res[o] : v;
            }
    return 0;
}
