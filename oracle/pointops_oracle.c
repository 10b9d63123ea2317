/*
 * oracle/pointops_oracle.c -- CPU restatement of the reference's point-cloud operator
 * hot path.  TEST INFRASTRUCTURE ONLY: nothing under toothgroupnetwork_b200/ may
 * import, link or execute this file.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs use it, and only as the checker
 * or as the timed CPU baseline.
 *
 * Parity status: the reference ships no tests and no golden vectors (SURVEY.md 4),
 * so this restatement is pinned against OUTPUTS OF THE REFERENCE ITSELF:
 *   - the reference CUDA kernels compiled verbatim for the GPU (oracle/_ref,
 *     built by oracle/Makefile) run on the GPU -> tests/golden/ref_cuda_*.npz
 *     (generator: tests/golden/make_ref_cuda_golden.py);
 *   - the reference's pure-torch pointnet2_utils functions imported from
 *     /root/reference on CPU -> tests/golden/ref_torch_*.npz
 *     (generator: tests/golden/make_ref_torch_golden.py).
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/external_libs).
 *
 * Build: gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC (see oracle/Makefile).
 * -ffp-contract=off matters: every fused multiply-add below is spelled fmaf() so the
 * rounding sequence is exactly the one the reference's SASS performs.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>

/* ---------------------------------------------------------------------------------
 * Launch-shape helper.  pointops/src/cuda_utils.h:11-14: block size is
 * 2^floor(log2(n)) capped to [1, 1024], with the log taken in double precision and
 * truncated -- reproduced literally because the FPS tie-break depends on it.
 * ------------------------------------------------------------------------------- */
int oracle_opt_n_threads(int work_size)
{
    const int p = (int)(log((double)work_size) / log(2.0));
    int t = 1 << p;
    if (t > 1024) t = 1024;
    if (t < 1) t = 1;
    return t;
}

/* Squared distance exactly as the reference's FPS / kNN kernels evaluate it after nvcc
 * contraction (pointops/src/sampling/sampling_cuda_kernel.cu:55,
 * knnquery/knnquery_cuda_kernel.cu:96; SASS: FMUL dy*dy, FFMA dx*dx+., FFMA dz*dz+.). */
static inline float sq_dist_fma(float ax, float ay, float az, float bx, float by, float bz)
{
    const float dx = bx - ax, dy = by - ay, dz = bz - az;
    float t = dy * dy;
    t = fmaf(dx, dx, t);
    return fmaf(dz, dz, t);
}

/* ---------------------------------------------------------------------------------
 * Farthest point sampling.  pointops/src/sampling/sampling_cuda_kernel.cu:14-129
 * (kernel), :131-171 (launcher).  One "block" of BS emulated threads per cloud:
 *   - idx[start_m] = start_n (:39);
 *   - each iteration: thread tid walks k = start_n+tid, +BS, ... keeping the running
 *     minimum in tmp[k] (:56-57) and its own first strict maximum (:58-59);
 *   - shared-memory tree over BS entries where the lower entry wins ties (:5-10,
 *     :64-123);
 *   - old = dists_i[0] (:125).
 * tmp must be pre-filled by the caller (the reference fills it with 1e10,
 * pointops/functions/pointops.py:22) and holds the final running minima on return.
 * ------------------------------------------------------------------------------- */
void oracle_furthestsampling(int b, int n_max, const float *xyz, const int *offset,
                             const int *new_offset, float *tmp, int *idx)
{
    const int bs = oracle_opt_n_threads(n_max);
    float *best = (float *)malloc(sizeof(float) * (size_t)bs);
    int *besti = (int *)malloc(sizeof(int) * (size_t)bs);
    for (int c = 0; c < b; ++c) {
        const int start_n = c ? offset[c - 1] : 0, end_n = offset[c];
        const int start_m = c ? new_offset[c - 1] : 0, end_m = new_offset[c];
        int old = start_n;
        if (start_m < end_m) idx[start_m] = start_n;             /* :39 */
        for (int j = start_m + 1; j < end_m; ++j) {
            for (int t = 0; t < bs; ++t) { best[t] = -1.0f; besti[t] = start_n; }
            const float ox = xyz[3 * (size_t)old], oy = xyz[3 * (size_t)old + 1], oz = xyz[3 * (size_t)old + 2];
            int t = 0;
            for (int k = start_n; k < end_n; ++k) {
                const float d = sq_dist_fma(ox, oy, oz, xyz[3 * (size_t)k], xyz[3 * (size_t)k + 1], xyz[3 * (size_t)k + 2]);
                const float d2 = d < tmp[k] ? d : tmp[k];            /* min(d, tmp[k]) */
                tmp[k] = d2;
                if (d2 > best[t]) { best[t] = d2; besti[t] = k; }     /* strict > */
                if (++t == bs) t = 0;
            }
            for (int s = bs >> 1; s >= 1; s >>= 1)
                for (int u = 0; u < s; ++u)
                    if (best[u + s] > best[u]) { best[u] = best[u + s]; besti[u] = besti[u + s]; }
            old = besti[0];
            idx[j] = old;
        }
    }
    free(best);
    free(besti);
}

/* ---------------------------------------------------------------------------------
 * k nearest neighbours inside the query's own segment.
 * pointops/src/knnquery/knnquery_cuda_kernel.cu:65-108; heap helpers :21-48;
 * segment lookup :51-62.  A size-k binary max-heap seeded with (1e10, start); a point
 * replaces the root only when strictly closer (:97); the heap is then sorted ascending
 * in place by repeated root extraction (:39-48).  The sift-down is restated with the
 * reference's exact comparison directions because the output order among equal
 * distances, and which of several equidistant points survive, depend on it.
 * dist2 receives SQUARED distances (the sqrt is taken in Python, pointops.py:43).
 * ------------------------------------------------------------------------------- */
static void sift_down(float *d, int *id, int len)
{
    int parent = 0;
    for (;;) {
        int kid = 2 * parent + 1;
        if (kid >= len) return;
        if (kid + 1 < len && d[kid + 1] > d[kid]) ++kid;
        if (d[parent] > d[kid]) return;
        const float fd = d[parent]; d[parent] = d[kid]; d[kid] = fd;
        const int fi = id[parent]; id[parent] = id[kid]; id[kid] = fi;
        parent = kid;
    }
}

void oracle_knnquery(int m, int nsample, const float *xyz, const float *new_xyz,
                     const int *offset, const int *new_offset, int *idx, float *dist2)
{
#pragma omp parallel
    {
        float *hd = (float *)malloc(sizeof(float) * (size_t)(nsample > 0 ? nsample : 1));
        int *hi = (int *)malloc(sizeof(int) * (size_t)(nsample > 0 ? nsample : 1));
#pragma omp for schedule(dynamic, 64)
        for (int q = 0; q < m; ++q) {
            int seg = 0;
            while (q >= new_offset[seg]) ++seg;                      /* :51-62 */
            const int start = seg ? offset[seg - 1] : 0, end = offset[seg];
            const float qx = new_xyz[3 * (size_t)q], qy = new_xyz[3 * (size_t)q + 1], qz = new_xyz[3 * (size_t)q + 2];
            for (int i = 0; i < nsample; ++i) { hd[i] = 1e10f; hi[i] = start; }
            for (int i = start; i < end; ++i) {
                /* the kernel writes (new - x); squares make the sign irrelevant */
                const float d = sq_dist_fma(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], qx, qy, qz);
                if (d < hd[0]) { hd[0] = d; hi[0] = i; sift_down(hd, hi, nsample); }
            }
            for (int last = nsample - 1; last > 0; --last) {         /* :39-48 */
                const float fd = hd[0]; hd[0] = hd[last]; hd[last] = fd;
                const int fi = hi[0]; hi[0] = hi[last]; hi[last] = fi;
                sift_down(hd, hi, last);
            }
            for (int i = 0; i < nsample; ++i) {
                idx[(size_t)q * nsample + i] = hi[i];
                dist2[(size_t)q * nsample + i] = hd[i];
            }
        }
        free(hd);
        free(hi);
    }
}

/* ---------------------------------------------------------------------------------
 * Gather / scatter family (pointops/src/{grouping,interpolation,subtraction,
 * aggregation}/*_cuda_kernel.cu).  The reference backward kernels accumulate with
 * fp32 atomicAdd in an unspecified order; the restatement accumulates in index order,
 * so backward parity is tested with a tolerance, forward parity bit-exactly.
 * ------------------------------------------------------------------------------- */

/* grouping_cuda_kernel.cu:5-14: out[m,k,c] = in[idx[m,k], c] */
void oracle_grouping_forward(int m, int nsample, int c, const float *in, const int *idx, float *out)
{
    for (size_t g = 0; g < (size_t)m * nsample; ++g)
        memcpy(out + g * c, in + (size_t)idx[g] * c, sizeof(float) * (size_t)c);
}

/* grouping_cuda_kernel.cu:16-25: grad_in[idx[m,k], c] += grad_out[m,k,c] (grad_in pre-zeroed) */
void oracle_grouping_backward(int m, int nsample, int c, const float *grad_out, const int *idx, float *grad_in)
{
    for (size_t g = 0; g < (size_t)m * nsample; ++g)
        for (int ch = 0; ch < c; ++ch) grad_in[(size_t)idx[g] * c + ch] += grad_out[g * c + ch];
}

/* interpolation_cuda_kernel.cu:5-18: out[n,c] += sum_k in[idx[n,k],c] * w[n,k], in k order
 * (out pre-zeroed by the caller; each term is a separate multiply then add -> nvcc
 * contracts "out += a*b" into fma(a, b, out)). */
void oracle_interpolation_forward(int n, int c, int k, const float *in, const int *idx, const float *w, float *out)
{
    for (int p = 0; p < n; ++p)
        for (int ch = 0; ch < c; ++ch) {
            float acc = out[(size_t)p * c + ch];
            for (int i = 0; i < k; ++i)
                acc = fmaf(in[(size_t)idx[(size_t)p * k + i] * c + ch], w[(size_t)p * k + i], acc);
            out[(size_t)p * c + ch] = acc;
        }
}

/* interpolation_cuda_kernel.cu:20-33 */
void oracle_interpolation_backward(int n, int c, int k, const float *grad_out, const int *idx, const float *w, float *grad_in)
{
    for (int p = 0; p < n; ++p)
        for (int ch = 0; ch < c; ++ch)
            for (int i = 0; i < k; ++i)
                grad_in[(size_t)idx[(size_t)p * k + i] * c + ch] += grad_out[(size_t)p * c + ch] * w[(size_t)p * k + i];
}

/* subtraction_cuda_kernel.cu:5-16: out[n,k,c] = in1[n,c] - in2[idx[n,k],c] */
void oracle_subtraction_forward(int n, int nsample, int c, const float *in1, const float *in2, const int *idx, float *out)
{
    for (int p = 0; p < n; ++p)
        for (int s = 0; s < nsample; ++s) {
            const size_t src = (size_t)idx[(size_t)p * nsample + s] * c;
            for (int ch = 0; ch < c; ++ch)
                out[((size_t)p * nsample + s) * c + ch] = in1[(size_t)p * c + ch] - in2[src + ch];
        }
}

/* subtraction_cuda_kernel.cu:18-30 */
void oracle_subtraction_backward(int n, int nsample, int c, const int *idx, const float *grad_out, float *grad_in1, float *grad_in2)
{
    for (int p = 0; p < n; ++p)
        for (int s = 0; s < nsample; ++s) {
            const size_t src = (size_t)idx[(size_t)p * nsample + s] * c;
            for (int ch = 0; ch < c; ++ch) {
                const float g = grad_out[((size_t)p * nsample + s) * c + ch];
                grad_in1[(size_t)p * c + ch] += g;
                grad_in2[src + ch] += -g;
            }
        }
}

/* aggregation_cuda_kernel.cu:5-20:
 * out[n,c] += sum_s (in[idx[n,s],c] + pos[n,s,c]) * w[n,s,c % w_c]   (contracted to fma) */
void oracle_aggregation_forward(int n, int nsample, int c, int w_c, const float *in, const float *pos,
                                const float *w, const int *idx, float *out)
{
    for (int p = 0; p < n; ++p)
        for (int ch = 0; ch < c; ++ch) {
            float acc = out[(size_t)p * c + ch];
            for (int s = 0; s < nsample; ++s) {
                const size_t g = (size_t)p * nsample + s;
                const float v = in[(size_t)idx[g] * c + ch] + pos[g * c + ch];
                acc = fmaf(v, w[g * w_c + ch % w_c], acc);
            }
            out[(size_t)p * c + ch] = acc;
        }
}

/* aggregation_cuda_kernel.cu:22-39 */
void oracle_aggregation_backward(int n, int nsample, int c, int w_c, const float *in, const float *pos,
                                 const float *w, const int *idx, const float *grad_out,
                                 float *grad_in, float *grad_pos, float *grad_w)
{
    for (int p = 0; p < n; ++p)
        for (int ch = 0; ch < c; ++ch)
            for (int s = 0; s < nsample; ++s) {
                const size_t g = (size_t)p * nsample + s;
                const size_t src = (size_t)idx[g] * c + ch;
                const float go = grad_out[(size_t)p * c + ch];
                const float wv = w[g * w_c + ch % w_c];
                grad_in[src] += go * wv;
                grad_pos[g * c + ch] = go * wv;
                grad_w[g * w_c + ch % w_c] += go * (in[src] + pos[g * c + ch]);
            }
}

/* ---------------------------------------------------------------------------------
 * PointNet++ side (pointnet2_utils/pointnet2_utils.py).  The reference computes the
 * pairwise distance in EXPANDED form through a K=3 matmul and two broadcast adds
 * (:36-41).  Probed against torch-CPU (MKL) in this container on 2.46e7 pairs: the
 * matmul is a k-sequential fma chain and the row sums are (x*x+y*y)+z*z unfused, i.e.
 *      d = -2 * fma(az,bz, fma(ay,by, ax*bx));  d += |a|^2;  d += |b|^2
 * bit for bit (tests/golden pins this with ref_torch_*.npz).
 * ------------------------------------------------------------------------------- */
static inline float sq_norm_torch(float x, float y, float z) { return (x * x + y * y) + z * z; }

static inline float sq_dist_expanded(float ax, float ay, float az, float an,
                                     float bx, float by, float bz, float bn)
{
    float dot = ax * bx;
    dot = fmaf(ay, by, dot);
    dot = fmaf(az, bz, dot);
    float d = -2.0f * dot;
    d += an;     /* src (first argument of square_distance) norm is added first (:39) */
    d += bn;
    return d;
}

/* square_distance, pointnet2_utils.py:20-41. src (n,3), dst (m,3) -> out (n,m) */
void oracle_square_distance(int n, int m, const float *src, const float *dst, float *out)
{
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        const float ax = src[3 * (size_t)i], ay = src[3 * (size_t)i + 1], az = src[3 * (size_t)i + 2];
        const float an = sq_norm_torch(ax, ay, az);
        for (int j = 0; j < m; ++j) {
            const float bx = dst[3 * (size_t)j], by = dst[3 * (size_t)j + 1], bz = dst[3 * (size_t)j + 2];
            out[(size_t)i * m + j] = sq_dist_expanded(ax, ay, az, an, bx, by, bz, sq_norm_torch(bx, by, bz));
        }
    }
}

/* query_ball_point, pointnet2_utils.py:120-144, one cloud: the first `nsample` indices in
 * ascending order whose expanded distance is NOT > r2 (r2 = float32(radius**2), the
 * scalar torch compares against), padded with the first hit; a query with no hit gets
 * the sentinel n in every slot exactly as the sort-and-mask formulation leaves it. */
void oracle_query_ball_point(int n, int s, float r2, int nsample, const float *xyz, const float *new_xyz, int64_t *group_idx)
{
#pragma omp parallel for schedule(dynamic, 16)
    for (int q = 0; q < s; ++q) {
        const float ax = new_xyz[3 * (size_t)q], ay = new_xyz[3 * (size_t)q + 1], az = new_xyz[3 * (size_t)q + 2];
        const float an = sq_norm_torch(ax, ay, az);
        int64_t *row = group_idx + (size_t)q * nsample;
        int cnt = 0;
        for (int j = 0; j < n && cnt < nsample; ++j) {
            const float bx = xyz[3 * (size_t)j], by = xyz[3 * (size_t)j + 1], bz = xyz[3 * (size_t)j + 2];
            const float d = sq_dist_expanded(ax, ay, az, an, bx, by, bz, sq_norm_torch(bx, by, bz));
            if (!(d > r2)) row[cnt++] = j;
        }
        const int64_t pad = cnt ? row[0] : (int64_t)n;
        for (; cnt < nsample; ++cnt) row[cnt] = pad;
    }
}

/* 3 nearest coarse points for PointNetFeaturePropagation, pointnet2_utils.py:333-335:
 * expanded distances, ascending; ties resolved towards the lower index (what a stable
 * sort gives; torch.sort is not documented stable, so tests mask exact ties).
 * xyz1 (n,3) fine, xyz2 (s,3) coarse -> dist (n,3), idx (n,3).  Requires s >= 3. */
void oracle_three_nn(int n, int s, const float *xyz1, const float *xyz2, float *dist, int64_t *idx)
{
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        const float ax = xyz1[3 * (size_t)i], ay = xyz1[3 * (size_t)i + 1], az = xyz1[3 * (size_t)i + 2];
        const float an = sq_norm_torch(ax, ay, az);
        float d0 = INFINITY, d1 = INFINITY, d2 = INFINITY;
        int i0 = 0, i1 = 0, i2 = 0;
        for (int j = 0; j < s; ++j) {
            const float bx = xyz2[3 * (size_t)j], by = xyz2[3 * (size_t)j + 1], bz = xyz2[3 * (size_t)j + 2];
            const float d = sq_dist_expanded(ax, ay, az, an, bx, by, bz, sq_norm_torch(bx, by, bz));
            if (d < d0) { d2 = d1; i2 = i1; d1 = d0; i1 = i0; d0 = d; i0 = j; }
            else if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = j; }
            else if (d < d2) { d2 = d; i2 = j; }
        }
        dist[3 * (size_t)i] = d0; dist[3 * (size_t)i + 1] = d1; dist[3 * (size_t)i + 2] = d2;
        idx[3 * (size_t)i] = i0; idx[3 * (size_t)i + 1] = i1; idx[3 * (size_t)i + 2] = i2;
    }
}

/* The reference's only CPU-capable FPS formulation (pointnet2_utils.py:72-86 /
 * :103-118, torch loop): direct (x-c)^2 summed over the last axis, update where
 * dist < distance, argmax = first maximum.  `start` replaces the random start (:109).
 * Used ONLY as the timed CPU baseline leg (cpu_baseline.kind == "port"). */
void oracle_fps_torchloop(int n, int npoint, int start, const float *xyz, float *distance, int64_t *centroids)
{
    int far = start;
    for (int j = 0; j < n; ++j) distance[j] = 1e10f;
    for (int i = 0; i < npoint; ++i) {
        centroids[i] = far;
        const float cx = xyz[3 * (size_t)far], cy = xyz[3 * (size_t)far + 1], cz = xyz[3 * (size_t)far + 2];
        float best = -INFINITY; int besti = 0;
        for (int j = 0; j < n; ++j) {
            const float dx = xyz[3 * (size_t)j] - cx, dy = xyz[3 * (size_t)j + 1] - cy, dz = xyz[3 * (size_t)j + 2] - cz;
            const float d = (dx * dx + dy * dy) + dz * dz;
            if (d < distance[j]) distance[j] = d;
            if (distance[j] > best) { best = distance[j]; besti = j; }
        }
        far = besti;
    }
}

/* Sampling + neighbour search of one set-abstraction level for a batch of clouds, one cloud per
 * OpenMP thread: the reference's CPU-capable FPS loop (pointnet2_utils.py:103-118, start 0),
 * the gather of the sampled centres (:157) and query_ball_point (:120-144).  This is the host
 * baseline bench.py times; the inner routines run serially inside each thread. */
void oracle_sa_sample_and_search_batch(int B, int n, int npoint, float r2, int nsample, const float *xyz,
                                       int64_t *fps, float *new_xyz, int64_t *group_idx)
{
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < B; ++b) {
        const float *cx = xyz + (size_t)b * n * 3;
        int64_t *cf = fps + (size_t)b * npoint;
        float *cn = new_xyz + (size_t)b * npoint * 3;
        float *dist = (float *)malloc(sizeof(float) * (size_t)n);
        oracle_fps_torchloop(n, npoint, 0, cx, dist, cf);
        free(dist);
        for (int s = 0; s < npoint; ++s) memcpy(cn + 3 * (size_t)s, cx + 3 * (size_t)cf[s], 3 * sizeof(float));
        oracle_query_ball_point(n, npoint, r2, nsample, cx, cn, group_idx + (size_t)b * npoint * nsample);
    }
}

/* Grouped shared MLP + max of one set-abstraction level for a batch of clouds, one cloud per OpenMP thread
 * (PointNetSetAbstraction.forward pointnet2_utils.py:227-237 with eval-mode BatchNorm): for every sampled centre s
 * gather its K neighbours as rows [xyz - centre | feats] (:163-169), run L x (1x1 conv + BatchNorm + ReLU) on the
 * (K, C) tile while it is cache-resident, keep the max over the K rows.  Weights arrive TRANSPOSED (wt[l]: (C_l, C_{l+1})
 * row-major) with BatchNorm given as per-channel scale / shift applied after the convolution (y = scale*(Wx) + shift,
 * shift already holding scale*bias), so that the inner loop is a vectorisable axpy over output channels.
 * This is the CPU baseline's MLP leg (bench.py) -- contiguous tiles, per-cloud threads: it scales with cores, unlike
 * running the reference's permuted (B,C,K,S) tensor through whole-tensor passes. */
__attribute__((target_clones("arch=skylake-avx512", "arch=haswell", "default")))
static void sa_mlp_max_cloud(int n, int S, int K, int D, const float *xyz, const float *feats, const float *new_xyz,
                             const int64_t *gidx, int L, const int *ch, const float *const *wt, const float *const *scale,
                             const float *const *shift, float *out /* (C_out, S) */, float *buf0, float *buf1)
{
    const int c0 = ch[0], cl = ch[L];
    for (int s = 0; s < S; ++s) {
        float *x = buf0, *y = buf1;
        for (int k = 0; k < K; ++k) {
            const int64_t j = gidx[(size_t)s * K + k];
            float *row = x + (size_t)k * c0;
            if (j < 0 || j >= n) { for (int c = 0; c < c0; ++c) row[c] = 0.f; continue; }
            for (int a = 0; a < 3; ++a) row[a] = xyz[3 * (size_t)j + a] - new_xyz[3 * (size_t)s + a];
            for (int d = 0; d < D; ++d) row[3 + d] = feats[(size_t)j * D + d];
        }
        for (int l = 0; l < L; ++l) {
            const int ci = ch[l], co = ch[l + 1];
            const float *w = wt[l], *sc = scale[l], *sh = shift[l];
            for (int k = 0; k < K; ++k) {
                const float *xi = x + (size_t)k * ci;
                float *yo = y + (size_t)k * co;
                for (int o = 0; o < co; ++o) yo[o] = 0.f;
                for (int c = 0; c < ci; ++c) {
                    const float xv = xi[c];
                    const float *wr = w + (size_t)c * co;
                    for (int o = 0; o < co; ++o) yo[o] += xv * wr[o];
                }
                for (int o = 0; o < co; ++o) {
                    const float v = yo[o] * sc[o] + sh[o];
                    yo[o] = v > 0.f ? v : 0.f;
                }
            }
            float *t = x; x = y; y = t;
        }
        for (int o = 0; o < cl; ++o) {
            float m = x[o];
            for (int k = 1; k < K; ++k) { const float v = x[(size_t)k * cl + o]; m = v > m ? v : m; }
            out[(size_t)o * S + s] = m;
        }
    }
}

void oracle_sa_group_mlp_max_batch(int B, int n, int S, int K, int D, const float *xyz, const float *feats,
                                   const float *new_xyz, const int64_t *gidx, int L, const int *ch,
                                   const float *const *wt, const float *const *scale, const float *const *shift, float *out)
{
    int cmax = 0;
    for (int l = 0; l <= L; ++l) cmax = ch[l] > cmax ? ch[l] : cmax;
#pragma omp parallel
    {
        float *buf0 = (float *)malloc(sizeof(float) * (size_t)K * cmax), *buf1 = (float *)malloc(sizeof(float) * (size_t)K * cmax);
#pragma omp for schedule(dynamic, 1)
        for (int b = 0; b < B; ++b)
            sa_mlp_max_cloud(n, S, K, D, xyz + (size_t)b * n * 3, feats ? feats + (size_t)b * n * D : NULL,
                             new_xyz + (size_t)b * S * 3, gidx + (size_t)b * S * K, L, ch, wt, scale, shift,
                             out + (size_t)b * ch[L] * S, buf0, buf1);
        free(buf0);
        free(buf1);
    }
}
