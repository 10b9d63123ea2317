/* dgcnn_knn_oracle.c -- CPU restatement of DGCNN's feature-space kNN (models/modules/dgcnn.py:4-10) as torch evaluates it on the
 * H100 (DESIGN §3.11).  TEST INFRASTRUCTURE ONLY: the checker of csrc/knn_feat.cu, written independently of it.
 * Compile with -ffp-contract=off: every operation below is rounded where it is written.
 *
 *   dot_ij = +0, then fmaf(x_ic, x_jc, dot) for c = 0..C-1              (cuBLAS FP32 GEMM, pinned by scripts/diag_dgcnn_knn.py)
 *   v_ij   = ((-xx_j) - (-2*dot_ij)) - xx_i                            (the reference's two element-wise subtractions)
 *   selection: the k largest by topk's radix key (-0 < +0, NaN largest), lower index first among equal keys
 *   order: the selection in gather order (entries above the k-th key by index, then those equal to it by index), sorted by
 *          at::native::bitonicSort<32> with the comparator GTOp<float, true>, thread by thread. */
#include <math.h>
#include <stdint.h>
#include <string.h>

static uint32_t radix_key(float v)
{
    uint32_t b;
    memcpy(&b, &v, 4);
    if (v != v) return 0xffffffffu;
    return b ^ ((b & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}

static int gt_nan(float a, float b) { return (isnan(a) && !isnan(b)) || a > b; }

static void bitonic_swap(float *ka, long long *va, int *oka, float *kb, long long *vb, int *okb, int dir)
{
    int swap = (gt_nan(*ka, *kb) && *oka) || !*okb;
    if (swap == dir) {
        float tk = *ka; *ka = *kb; *kb = tk;
        long long tv = *va; *va = *vb; *vb = tv;
        int to = *oka; *oka = *okb; *okb = to;
    }
}

/* at::native::bitonicSort with Power2SortSize = 32: 16 threads, each step applied for every thread in turn (the threads of one
 * step touch disjoint pairs, so the serial order is immaterial) */
static void bitonic_sort32(float *k, long long *v, int *ok)
{
    for (unsigned size = 2; size < 32; size *= 2)
        for (unsigned stride = size / 2; stride > 0; stride /= 2)
            for (unsigned t = 0; t < 16; ++t) {
                int flag = (t & (size / 2)) != 0;
                unsigned pos = 2 * t - (t & (stride - 1));
                bitonic_swap(k + pos, v + pos, ok + pos, k + pos + stride, v + pos + stride, ok + pos + stride, flag);
            }
    for (unsigned stride = 16; stride > 0; stride /= 2)
        for (unsigned t = 0; t < 16; ++t) {
            unsigned pos = 2 * t - (t & (stride - 1));
            bitonic_swap(k + pos, v + pos, ok + pos, k + pos + stride, v + pos + stride, ok + pos + stride, 0);
        }
}

static float dot_product(const float *xb, int N, int C, int i, int j)
{
    float dot = 0.0f;
    for (int c = 0; c < C; ++c) dot = fmaf(xb[(long long)c * N + i], xb[(long long)c * N + j], dot);
    return dot;
}

/* x (B, C, N) contiguous, xx (B, N); idx (B, N, k) int64, val (B, N, k) float32.  1 <= k <= 32, k <= N. */
void oracle_dgcnn_knn(int B, int N, int C, int k, const float *x, const float *xx, long long *idx, float *val)
{
    for (int b = 0; b < B; ++b) {
        const float *xb = x + (long long)b * C * N, *xxb = xx + (long long)b * N;
#pragma omp parallel for schedule(dynamic, 16)
        for (int i = 0; i < N; ++i) {
            uint32_t lk[32];
            int li[32], cnt = 0;
            for (int j = 0; j < N; ++j) {
                const float dot = dot_product(xb, N, C, i, j);
                const float inner = -2.0f * dot;
                const float t = (-xxb[j]) - inner;
                const float v = t - xxb[i];
                const uint32_t key = radix_key(v);
                /* j ascends, so among equal keys the earlier entry keeps its place */
                if (cnt == k && key <= lk[k - 1]) continue;
                int p = cnt < k ? cnt : k - 1;
                while (p > 0 && lk[p - 1] < key) { lk[p] = lk[p - 1]; li[p] = li[p - 1]; --p; }
                lk[p] = key;
                li[p] = j;
                if (cnt < k) ++cnt;
            }
            /* gather order */
            const uint32_t kth = lk[k - 1];
            float sk[32];
            long long sv[32];
            int ok[32], g = 0;
            for (int j = 0; j < N && g < k; ++j)
                for (int e = 0; e < k; ++e)
                    if (li[e] == j && lk[e] > kth) { sv[g] = j; g++; }
            for (int e = 0; e < k; ++e)
                if (lk[e] == kth) sv[g++] = li[e];
            for (int e = 0; e < 32; ++e) {
                ok[e] = e < k;
                if (e >= k) { sk[e] = 0.0f; sv[e] = 0; continue; }
                const long long j = sv[e];
                sk[e] = ((-xxb[j]) - (-2.0f * dot_product(xb, N, C, i, (int)j))) - xxb[i];
            }
            if (k > 1) bitonic_sort32(sk, sv, ok);
            for (int e = 0; e < k; ++e) {
                idx[((long long)b * N + i) * k + e] = sv[e];
                val[((long long)b * N + i) * k + e] = sk[e];
            }
        }
    }
}
