// fps.cu -- farthest point sampling for sm_90a.
//
// Replaces pointops/src/sampling/sampling_cuda_kernel.cu:14-171 of the reference (one CTA per
// cloud re-streaming xyz+tmp from L2 every iteration, 11 block barriers per iteration).
//
// Design (DESIGN.md "FPS"):
//  * A thread-block CLUSTER of CS CTAs owns G clouds at a time.  Every point (x,y,z and its
//    running minimum t) lives in REGISTERS for the whole kernel: thread u holds SLOTS points of
//    each cloud, packed two per 64-bit register so the distance update runs on
//    paired fp32 ops.  HBM is touched once to load the clouds and once per sample for idx.
//  * The argmax is tracked inside the update loop on the ALU pipe (FSETP/FMNMX/SEL run beside the
//    FP32 pipe, which is the bottleneck: 6 lane-ops per point-update), so no thread ever
//    re-scans its registers.
//  * Reduction is two-level and barrier-free: each warp reduces with two CREDUX ops and drops
//    one candidate in shared memory + arrives on a CTA-local mbarrier; one publisher warp per
//    cloud picks the CTA's candidate and sends (t, key, x, y, z, j) to the mailbox of every CTA of
//    the cluster with st.async, which also completes bytes on that CTA's mbarrier.
//  * G > 1 software-pipelines independent clouds through the same cluster: the candidates of
//    cloud g travel while the SM updates cloud g+1, hiding the DSMEM/mbarrier round trip that
//    dominates a single serial FPS chain.
//  * Bit-exact tie-break.  The reference picks, among equal maxima, the point with the smallest
//    (bitrev(j mod BS), j div BS) where BS is ITS block size (cuda_utils.h:11-14) and j the
//    cloud-local index: thread tid scans j = tid, tid+BS, .. with a strict '>' (first maximum
//    wins) and the shared-memory tree lets the lower entry win ties, which orders threads by the
//    bit-reversed tid (sampling_cuda_kernel.cu:5-10,49-59,64-123).  Here thread u owns residue
//    r = u mod BS and the contiguous slot range [q*SLOTS, (q+1)*SLOTS) with q = u div BS; its own
//    scan is the same strict '>' in slot order, threads are ordered by (bitrev(r), q), and
//    candidates by the point key (bitrev(j mod BS), j div BS).
//  * Distance arithmetic is the reference's SASS sequence: t = dy*dy; t = fma(dx,dx,t);
//    d = fma(dz,dz,t); min; all IEEE-rn, so indices are bit-identical.
#include <algorithm>
#include <climits>
#include <cmath>

#include "common.cuh"
#include "fps.cuh"
#include "tgn_b200.h"

#include <cstdio>

namespace tgn {
namespace {

constexpr int kCandWords = 8;      // one mailbox entry = 32 bytes (24 used)
constexpr int kCandBytes = 24;     // bytes completed on the mbarrier per candidate

__device__ __forceinline__ int bitrev_low(int v, int bits) {
    return bits ? static_cast<int>(__brev(static_cast<unsigned>(v)) >> (32 - bits)) : 0;
}
// Total order of points under the reference's tie-break (smaller wins).
__device__ __forceinline__ int point_key(int j, int bs_log2) {
    return (bitrev_low(j & ((1 << bs_log2) - 1), bs_log2) << 21) | (j >> bs_log2);
}

template <int T, int SLOTS, int CS, int G>
__global__ void __launch_bounds__(T, 1)
fps_resident_kernel(const float* __restrict__ xyz, const int* __restrict__ offset,
                    const int* __restrict__ new_offset, float* tmp, int* __restrict__ idx, int b, int bs_log2)
{
    static_assert(SLOTS % 2 == 0, "slots are processed in packed pairs");
    constexpr int NW = T / 32;
    constexpr int PAIRS = SLOTS / 2;
    constexpr unsigned FULL = 0xffffffffu;

    __shared__ __align__(16) uint32_t mailbox[G][2][CS * kCandWords];   // one candidate per CTA of the cluster
    __shared__ __align__(16) uint32_t wslot[G][2][NW * 4];              // one candidate per warp of this CTA
    __shared__ __align__(8) uint64_t mbars[G][2];                       // mailbox full (cluster scope)
    __shared__ __align__(8) uint64_t lbars[G][2];                       // warp candidates full (CTA scope)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = (CS > 1) ? static_cast<int>(cluster_ctarank()) : 0;
    const int cluster = blockIdx.x / CS;

    int start_n[G], n[G], start_m[G], m[G];
    int mmax = 0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const int cloud = cluster * G + g;
        start_n[g] = 0; n[g] = 0; start_m[g] = 0; m[g] = 0;
        if (cloud < b) {
            start_n[g] = cloud ? __ldg(offset + cloud - 1) : 0;
            n[g] = __ldg(offset + cloud) - start_n[g];
            start_m[g] = cloud ? __ldg(new_offset + cloud - 1) : 0;
            m[g] = __ldg(new_offset + cloud) - start_m[g];
            if (n[g] <= 0) m[g] = 0;
            if (m[g] > 0 && rank == 0 && tid == 0) idx[start_m[g]] = start_n[g];   // sampling_cuda_kernel.cu:39
        }
        mmax = max(mmax, m[g]);
    }
    if (mmax <= 1) return;                              // uniform across the cluster

    if (tid == 0) {
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                mbar_init(smem_u32(&mbars[g][p]), 1);
                mbar_init(smem_u32(&lbars[g][p]), NW);
            }
        mbar_fence_init();
        if (CS > 1) {
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int p = 0; p < 2; ++p) mbar_arrive_expect_tx(smem_u32(&mbars[g][p]), CS * kCandBytes);
        }
    }
    if (CS > 1) cluster_sync_all(); else __syncthreads();

    // ---- load this thread's points into registers ------------------------------------------
    const int bs = 1 << bs_log2;
    const int u = rank * T + tid;
    const int r = u & (bs - 1);
    const int q = u >> bs_log2;
    const int tprio = (bitrev_low(r, bs_log2) << 14) | q;

    uint64_t X[G][PAIRS], Y[G][PAIRS], Z[G][PAIRS];
    float t[G][SLOTS];
    float ox[G], oy[G], oz[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const float* cxyz = xyz + 3 * static_cast<size_t>(start_n[g]);
        const float* ctmp = tmp ? tmp + start_n[g] : nullptr;
#pragma unroll
        for (int p = 0; p < PAIRS; ++p) {
            float c[2][3];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = (q * SLOTS + 2 * p + h) * bs + r;
                const bool ok = j < n[g] && m[g] > 1;
                c[h][0] = ok ? __ldg(cxyz + 3 * static_cast<size_t>(j) + 0) : 0.f;
                c[h][1] = ok ? __ldg(cxyz + 3 * static_cast<size_t>(j) + 1) : 0.f;
                c[h][2] = ok ? __ldg(cxyz + 3 * static_cast<size_t>(j) + 2) : 0.f;
                t[g][2 * p + h] = ok ? (ctmp ? ctmp[j] : 1e10f) : -1.0f;   // pads can never be a maximum
            }
            X[g][p] = pack2(c[0][0], c[1][0]);
            Y[g][p] = pack2(c[0][1], c[1][1]);
            Z[g][p] = pack2(c[0][2], c[1][2]);
        }
        const bool any = m[g] > 1;
        ox[g] = any ? __ldg(cxyz + 0) : 0.f;
        oy[g] = any ? __ldg(cxyz + 1) : 0.f;
        oz[g] = any ? __ldg(cxyz + 2) : 0.f;
    }

    // Winner of iteration `itp` of cloud g: wait for the mailbox, pick the best of the CS
    // candidates, record it.  Executed by every warp (each needs the coordinates).
    auto consume = [&](int g, int itp) {
        const int par = itp & 1;
        const uint32_t bar = smem_u32(&mbars[g][par]);
        mbar_wait(bar, ((itp - 1) >> 1) & 1);
        int cv = INT_MIN, ck = INT_MAX;
        if (lane < CS) {
            const uint2 vk = *reinterpret_cast<const uint2*>(&mailbox[g][par][lane * kCandWords]);
            cv = static_cast<int>(vk.x);
            ck = static_cast<int>(vk.y);
        }
        int src = 0;
        if (CS > 1) {
            const int gmax = __reduce_max_sync(FULL, cv);
            const int gkey = __reduce_min_sync(FULL, cv == gmax ? ck : INT_MAX);
            src = __ffs(__ballot_sync(FULL, cv == gmax && ck == gkey)) - 1;
        }
        const uint4 w0 = *reinterpret_cast<const uint4*>(&mailbox[g][par][src * kCandWords]);
        const uint2 w1 = *reinterpret_cast<const uint2*>(&mailbox[g][par][src * kCandWords + 4]);
        ox[g] = __uint_as_float(w0.z);
        oy[g] = __uint_as_float(w0.w);
        oz[g] = __uint_as_float(w1.x);
        if (warp == g % NW && lane == 0) {
            if (rank == 0) idx[start_m[g] + itp] = start_n[g] + static_cast<int>(w1.y);
            // Re-arm this parity for iteration itp+2 before this warp publishes itp+1: nobody can
            // complete bytes on that phase before receiving this CTA's candidate of itp+1.
            if (CS > 1 && itp + 2 < m[g]) mbar_arrive_expect_tx(bar, CS * kCandBytes);
        }
    };

    for (int it = 1; it < mmax; ++it) {
        const int par = it & 1;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            if (it >= m[g]) continue;
            if (it > 1) consume(g, it - 1);

            // ---- update the running minima of cloud g and track this thread's first maximum ----
            const uint64_t OX = pack2(ox[g], ox[g]), OY = pack2(oy[g], oy[g]), OZ = pack2(oz[g], oz[g]);
            float best = -1.0f;
            int bsel = 0;
#pragma unroll
            for (int p = 0; p < PAIRS; ++p) {
                const uint64_t dx = sub2(X[g][p], OX), dy = sub2(Y[g][p], OY), dz = sub2(Z[g][p], OZ);
                uint64_t d = mul2(dy, dy);
                d = fma2(dx, dx, d);
                d = fma2(dz, dz, d);
                float dl, dh;
                unpack2(d, dl, dh);
                const float ta = fminf(dl, t[g][2 * p]);
                t[g][2 * p] = ta;
                if (ta > best) { best = ta; bsel = 2 * p; }             // strict '>': first maximum wins
                const float tb = fminf(dh, t[g][2 * p + 1]);
                t[g][2 * p + 1] = tb;
                if (tb > best) { best = tb; bsel = 2 * p + 1; }
            }

            // ---- warp candidate: max value, then smallest thread priority among the tied lanes ----
            const int bi = __float_as_int(best);        // t >= 0 or -1: signed-int order == float order
            const int wmax = __reduce_max_sync(FULL, bi);
            const int wpri = __reduce_min_sync(FULL, bi == wmax ? tprio : INT_MAX);
            const uint32_t lbar = smem_u32(&lbars[g][par]);
            if (bi == wmax && tprio == wpri) {          // exactly one lane
                const int j = (q * SLOTS + bsel) * bs + r;
                *reinterpret_cast<uint4*>(&wslot[g][par][warp * 4]) =
                    make_uint4(static_cast<uint32_t>(bi), static_cast<uint32_t>(point_key(j, bs_log2)), static_cast<uint32_t>(j), 0u);
                mbar_arrive(lbar);                      // release.cta: the store above is visible to the waiter
            }

            // ---- publisher warp of cloud g: CTA candidate -> every CTA of the cluster -----------------
            if (warp == g % NW) {
                mbar_wait(lbar, ((it - 1) >> 1) & 1);
                int cv = INT_MIN, ck = INT_MAX, cj = 0;
                if (NW == 32 || lane < NW) {
                    const uint4 c = *reinterpret_cast<const uint4*>(&wslot[g][par][lane * 4]);
                    cv = static_cast<int>(c.x); ck = static_cast<int>(c.y); cj = static_cast<int>(c.z);
                }
                const int cmax = __reduce_max_sync(FULL, cv);
                const int ckey = __reduce_min_sync(FULL, cv == cmax ? ck : INT_MAX);
                const int src = __ffs(__ballot_sync(FULL, cv == cmax && ck == ckey)) - 1;
                const int jw = __shfl_sync(FULL, cj, src);
                if (lane == 0) {
                    // a CTA whose slice of a tiny cloud holds only pads publishes a losing candidate (value -1) whose index lies
                    // past the cloud: its coordinates are never used, but the read must stay inside the cloud
                    const float* pw = xyz + 3 * (static_cast<size_t>(start_n[g]) + (jw < n[g] ? jw : 0));
                    const float wx = __ldg(pw), wy = __ldg(pw + 1), wz = __ldg(pw + 2);
                    uint32_t* slot = &mailbox[g][par][rank * kCandWords];
                    if (CS > 1) {
                        const uint32_t sa = smem_u32(slot), ba = smem_u32(&mbars[g][par]);
#pragma unroll
                        for (int dst = 0; dst < CS; ++dst) {
                            const uint32_t ra = map_to_cta(sa, dst), rb = map_to_cta(ba, dst);
                            st_async_v4(ra, static_cast<uint32_t>(cmax), static_cast<uint32_t>(ckey), __float_as_uint(wx),
                                        __float_as_uint(wy), rb);
                            st_async_v2(ra + 16, __float_as_uint(wz), static_cast<uint32_t>(jw), rb);
                        }
                    } else {
                        *reinterpret_cast<uint4*>(slot) = make_uint4(static_cast<uint32_t>(cmax), static_cast<uint32_t>(ckey),
                                                                     __float_as_uint(wx), __float_as_uint(wy));
                        *reinterpret_cast<uint2*>(slot + 4) = make_uint2(__float_as_uint(wz), static_cast<uint32_t>(jw));
                        mbar_arrive(smem_u32(&mbars[g][par]));
                    }
                }
                __syncwarp();
            }
        }
    }
#pragma unroll
    for (int g = 0; g < G; ++g)
        if (m[g] > 1) consume(g, m[g] - 1);             // winner of the last iteration

    if (tmp) {
#pragma unroll
        for (int g = 0; g < G; ++g) {
            if (m[g] <= 1) continue;
            float* ctmp = tmp + start_n[g];
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) {
                const int j = (q * SLOTS + s) * bs + r;
                if (j < n[g]) ctmp[j] = t[g][s];
            }
        }
    }
    if (CS > 1) cluster_sync_all();   // no CTA leaves while a peer may still address its shared memory
}

// --------------------------------------------------------------------------------------------
// Streaming kernel for clouds that do not fit the register-resident kernels (n > 8*12288) or
// when a cluster cannot be scheduled: one CTA of 1024 threads per cloud, xyz and tmp re-read
// from L2 each iteration as in the reference, but with one barrier per iteration instead of
// eleven and the same exact tie-break.  tmp is required.
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1)
fps_stream_kernel(const float* __restrict__ xyz, const int* __restrict__ offset, const int* __restrict__ new_offset,
                  float* __restrict__ tmp, int* __restrict__ idx, int bs_log2)
{
    constexpr int T = 1024, NW = T / 32;
    constexpr unsigned FULL = 0xffffffffu;
    __shared__ int2 wbuf[2][NW];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const int start_n = cloud ? offset[cloud - 1] : 0;
    const int n = offset[cloud] - start_n;
    const int start_m = cloud ? new_offset[cloud - 1] : 0;
    const int m = new_offset[cloud] - start_m;
    if (m <= 0 || n <= 0) return;
    if (tid == 0) idx[start_m] = start_n;
    const int bs = 1 << bs_log2;
    const int r = tid & (bs - 1), q = tid >> bs_log2, chunks = T >> bs_log2;
    const int ns = (n + bs - 1) >> bs_log2;             // slots per residue
    const int spc = (ns + chunks - 1) / chunks;         // slots per chunk
    const int tprio = (bitrev_low(r, bs_log2) << 14) | q;
    const float* cxyz = xyz + 3 * static_cast<size_t>(start_n);
    float* ctmp = tmp + start_n;
    int old = 0;
    for (int it = 1; it < m; ++it) {
        const float ox = cxyz[3 * static_cast<size_t>(old)], oy = cxyz[3 * static_cast<size_t>(old) + 1],
                    oz = cxyz[3 * static_cast<size_t>(old) + 2];
        float best = -1.0f;
        int bj = 0;
        const int s_end = min((q + 1) * spc, ns);
        for (int sg = q * spc; sg < s_end; ++sg) {
            const int j = sg * bs + r;
            if (j < n) {
                const float dx = cxyz[3 * static_cast<size_t>(j)] - ox, dy = cxyz[3 * static_cast<size_t>(j) + 1] - oy,
                            dz = cxyz[3 * static_cast<size_t>(j) + 2] - oz;
                float d = __fmul_rn(dy, dy);
                d = __fmaf_rn(dx, dx, d);
                d = __fmaf_rn(dz, dz, d);
                const float v = fminf(d, ctmp[j]);
                ctmp[j] = v;
                if (v > best) { best = v; bj = j; }
            }
        }
        const int bi = __float_as_int(best);
        const int wmax = __reduce_max_sync(FULL, bi);
        const int wpri = __reduce_min_sync(FULL, bi == wmax ? tprio : INT_MAX);
        if (bi == wmax && tprio == wpri) wbuf[it & 1][warp] = make_int2(bi, bj);
        __syncthreads();
        const int2 c = wbuf[it & 1][lane];              // NW == 32: one candidate per lane
        const int key = point_key(c.y, bs_log2);
        const int gmax = __reduce_max_sync(FULL, c.x);
        const int gkey = __reduce_min_sync(FULL, c.x == gmax ? key : INT_MAX);
        const int src = __ffs(__ballot_sync(FULL, c.x == gmax && key == gkey)) - 1;
        old = __shfl_sync(FULL, c.y, src);
        if (tid == 0) idx[start_m + it] = start_n + old;
    }
}

// cuda_utils.h:11-14 of the reference, literally (double log, truncation).
int ref_block_log2(int n)
{
    const int p = static_cast<int>(std::log(static_cast<double>(n)) / std::log(2.0));
    int bs = std::max(std::min(1 << p, 1024), 1);
    int l = 0;
    while ((1 << l) < bs) ++l;
    return l;
}

template <int T, int SLOTS, int CS, int G>
int launch_resident(int b, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx,
                    int bs_log2, cudaStream_t stream)
{
    auto kern = fps_resident_kernel<T, SLOTS, CS, G>;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>((b + G - 1) / G) * CS);
    cfg.blockDim = dim3(T);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, xyz, offset, new_offset, tmp, idx, b, bs_log2);
    if (e != cudaSuccess) {
        set_error("fps_resident_kernel<%d,%d,%d,%d> launch failed: %s", T, SLOTS, CS, G, cudaGetErrorString(e));
        (void)cudaGetLastError();
        return TGN_ERR_CUDA;
    }
    return check_launch("fps_resident_kernel");
}

struct FpsConfig { int T, SLOTS, CS, G; };

// (T, SLOTS per cloud, cluster size, clouds in flight per cluster); register budget:
// 4 * SLOTS * G data registers per thread, 128 at T=512, 64 at T=1024.
const FpsConfig kConfigs[] = {
    {128, 4, 1, 1}, {256, 4, 1, 1}, {512, 4, 1, 1}, {1024, 4, 1, 1}, {1024, 8, 1, 1},
    {512, 4, 2, 1}, {512, 8, 2, 1}, {512, 12, 2, 1}, {512, 16, 2, 1}, {512, 24, 2, 1},
    {512, 4, 4, 1}, {512, 8, 4, 1}, {512, 12, 4, 1}, {512, 16, 4, 1}, {512, 24, 4, 1},
    {512, 4, 8, 1}, {512, 8, 8, 1}, {512, 12, 8, 1}, {512, 16, 8, 1}, {512, 24, 8, 1},
    // software-pipelined: two clouds per cluster
    {512, 4, 1, 2}, {512, 8, 1, 2}, {512, 12, 1, 2},
    {512, 4, 2, 2}, {512, 8, 2, 2}, {512, 12, 2, 2},
    {512, 4, 4, 2}, {512, 8, 4, 2}, {512, 12, 4, 2},
    {512, 8, 8, 2}, {512, 12, 8, 2},
};

// Smallest resident configuration that holds n_max points at cluster size cs with g clouds in flight.
FpsConfig pick_config(int n_max, int bs_log2, int cs, int g)
{
    const int bs = 1 << bs_log2;
    for (const FpsConfig& c : kConfigs) {
        if (c.CS != cs || c.G != g) continue;
        const int v = c.T * c.CS;
        if (v < bs) continue;
        const long long cap_slots = static_cast<long long>(v / bs) * c.SLOTS;     // slots per residue
        if (cap_slots >= (n_max + bs - 1) / bs) return c;
    }
    return {0, 0, 0, 0};
}

#define TGN_FPS_CASE(T_, S_, C_, G_)                                                                  \
    if (c.T == T_ && c.SLOTS == S_ && c.CS == C_ && c.G == G_)                                         \
        return launch_resident<T_, S_, C_, G_>(b, xyz, offset, new_offset, tmp, idx, bs_log2, stream);

int dispatch_resident(const FpsConfig& c, int b, const float* xyz, const int* offset, const int* new_offset,
                      float* tmp, int* idx, int bs_log2, cudaStream_t stream)
{
    TGN_FPS_CASE(128, 4, 1, 1) TGN_FPS_CASE(256, 4, 1, 1) TGN_FPS_CASE(512, 4, 1, 1) TGN_FPS_CASE(1024, 4, 1, 1)
    TGN_FPS_CASE(1024, 8, 1, 1)
    TGN_FPS_CASE(512, 4, 2, 1) TGN_FPS_CASE(512, 8, 2, 1) TGN_FPS_CASE(512, 12, 2, 1) TGN_FPS_CASE(512, 16, 2, 1)
    TGN_FPS_CASE(512, 24, 2, 1)
    TGN_FPS_CASE(512, 4, 4, 1) TGN_FPS_CASE(512, 8, 4, 1) TGN_FPS_CASE(512, 12, 4, 1) TGN_FPS_CASE(512, 16, 4, 1)
    TGN_FPS_CASE(512, 24, 4, 1)
    TGN_FPS_CASE(512, 4, 8, 1) TGN_FPS_CASE(512, 8, 8, 1) TGN_FPS_CASE(512, 12, 8, 1) TGN_FPS_CASE(512, 16, 8, 1)
    TGN_FPS_CASE(512, 24, 8, 1)
    TGN_FPS_CASE(512, 4, 1, 2) TGN_FPS_CASE(512, 8, 1, 2) TGN_FPS_CASE(512, 12, 1, 2)
    TGN_FPS_CASE(512, 4, 2, 2) TGN_FPS_CASE(512, 8, 2, 2) TGN_FPS_CASE(512, 12, 2, 2)
    TGN_FPS_CASE(512, 4, 4, 2) TGN_FPS_CASE(512, 8, 4, 2) TGN_FPS_CASE(512, 12, 4, 2)
    TGN_FPS_CASE(512, 8, 8, 2) TGN_FPS_CASE(512, 12, 8, 2)
    set_error("no resident FPS kernel for T=%d SLOTS=%d CS=%d G=%d", c.T, c.SLOTS, c.CS, c.G);
    return TGN_ERR_INVALID;
}

}  // namespace

// mode: 0 auto, -1 streaming kernel, -2 bucket-pruned kernel, otherwise 100*G + CS (G omitted = 1):
// force that register-resident shape.
int fps_dispatch(int b, int n_max, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx,
                 int mode, cudaStream_t stream)
{
    if (b <= 0) return TGN_OK;
    if (n_max <= 0) { set_error("furthestsampling: n_max must be positive"); return TGN_ERR_INVALID; }
    const int bs_log2 = ref_block_log2(n_max);
    if (mode == -1) {
        if (!tmp) { set_error("furthestsampling: the streaming kernel needs a tmp buffer"); return TGN_ERR_INVALID; }
        fps_stream_kernel<<<b, 1024, 0, stream>>>(xyz, offset, new_offset, tmp, idx, bs_log2);
        return check_launch("fps_stream_kernel");
    }
    // Auto: small clouds stay register-resident in one CTA (cheapest iteration); everything larger
    // goes to the bucket-pruned kernel, which wins both on latency and on throughput.
    // mode -2: bucket kernel, shape by batch size; mode -(10 + W): bucket kernel with W warps per cloud.
    // mode -3 / -(40 + W): the same with the single-barrier schedule (fps_bucket_kernel2).
    if (mode == -3 || (mode <= -41 && mode >= -72)) {
        if (n_max > fps_bucket_max_points()) { set_error("furthestsampling: n_max=%d exceeds the bucket kernel", n_max); return TGN_ERR_INVALID; }
        return fps_bucket_launch(b, n_max, xyz, offset, new_offset, tmp, idx, bs_log2, 100 + (mode == -3 ? 0 : -mode - 40), stream);
    }
    // mode -(80 + W): single barrier AND register-resident bucket tables (fps_bucket_kernel3; clouds with more buckets per lane
    // than the registers hold keep the tables in shared memory).
    if (mode <= -81 && mode >= -112) {
        if (n_max > fps_bucket_max_points()) { set_error("furthestsampling: n_max=%d exceeds the bucket kernel", n_max); return TGN_ERR_INVALID; }
        return fps_bucket_launch(b, n_max, xyz, offset, new_offset, tmp, idx, bs_log2, 200 + (-mode - 80), stream);
    }
    if (mode == -2 || (mode <= -11 && mode >= -26) || (mode == 0 && n_max > 4096 && n_max <= fps_bucket_max_points())) {
        if (n_max > fps_bucket_max_points()) { set_error("furthestsampling: n_max=%d exceeds the bucket kernel", n_max); return TGN_ERR_INVALID; }
        return fps_bucket_launch(b, n_max, xyz, offset, new_offset, tmp, idx, bs_log2, mode <= -11 ? -mode - 10 : 0, stream);
    }
    FpsConfig cfg{0, 0, 0, 0};
    if (mode > 0) {
        cfg = pick_config(n_max, bs_log2, mode % 100, std::max(1, mode / 100));
    } else {
        const int sms = sm_count();
        // Throughput shape: two clouds pipelined through the smallest cluster that holds them,
        // when there are at least two clouds and the batch can occupy the machine that way.
        // (the pipelined shapes lose to one cloud per 2-CTA cluster at
        //  24k points because per-warp reduction overhead doubles with the cluster size, so auto
        //  mode does not pick them; they stay reachable through `mode` for experiments)
        if (false && b >= 2) {
            for (int cs = 1; cs <= 8 && !cfg.T; cs *= 2) {
                const FpsConfig c = pick_config(n_max, bs_log2, cs, 2);
                if (c.T && static_cast<long long>((b + 1) / 2) * cs * 2 > sms / 2) cfg = c;
                else if (c.T) break;
            }
        }
        if (!cfg.T) {
            // Latency shape: one cloud per cluster, widened while SMs are idle and each CTA still
            // holds >= 1024 points.
            int first = 0;
            for (int cs = 1; cs <= 8; cs *= 2)
                if (pick_config(n_max, bs_log2, cs, 1).T) { first = cs; break; }
            if (first) {
                int cs = first;
                while (cs < 8 && static_cast<long long>(b) * cs * 2 <= sms && n_max / (cs * 2) >= 1024 &&
                       pick_config(n_max, bs_log2, cs * 2, 1).T)
                    cs *= 2;
                cfg = pick_config(n_max, bs_log2, cs, 1);
            }
        }
    }
    if (!cfg.T) {
        if (mode > 0) { set_error("furthestsampling: no resident kernel of shape %d for n_max=%d", mode, n_max); return TGN_ERR_INVALID; }
        if (!tmp) {
            set_error("furthestsampling: n_max=%d exceeds the register-resident kernels and no tmp buffer was given", n_max);
            return TGN_ERR_INVALID;
        }
        fps_stream_kernel<<<b, 1024, 0, stream>>>(xyz, offset, new_offset, tmp, idx, bs_log2);
        return check_launch("fps_stream_kernel");
    }
    return dispatch_resident(cfg, b, xyz, offset, new_offset, tmp, idx, bs_log2, stream);
}

}  // namespace tgn

extern "C" {

int tgn_furthestsampling(int b, int n_max, const float* xyz, const int* offset, const int* new_offset, float* tmp,
                         int* idx, int mode, void* stream)
{
    return tgn::fps_dispatch(b, n_max, xyz, offset, new_offset, tmp, idx, mode, static_cast<cudaStream_t>(stream));
}

void furthestsampling_cuda_launcher(int b, int n, const float* xyz, const int* offset, const int* new_offset, float* tmp,
                                    int* idx)
{
    // void like the reference's launcher: a rejected call is reported on stderr instead of returning silently
    if (tgn::fps_dispatch(b, n, xyz, offset, new_offset, tmp, idx, 0, static_cast<cudaStream_t>(0)) != TGN_OK)
        std::fprintf(stderr, "libtgn_b200: %s\n", tgn_last_error());
}

}  // extern "C"
