// meanshift.cu -- the seed ascent of scikit-learn 1.9's MeanShift(bandwidth).fit on float64 (n,3) points (seeds = X,
// cluster_all), one warp per seed, every seed in one launch (DESIGN §3.14).  The KD tree is scikit-learn's own
// KDTree(X, leaf_size=30), built on the host: its points in tree order (idx_array), node ranges, leaf flags and node bounds.
//
// Each mean update is _mean_shift_single_seed's: radius_neighbors returns the points with the float64 reduced distance
// ((0 + dx*dx) + dy*dy) + dz*dz <= r*r in ascending tree position, np.mean(axis=0) adds them in that order starting from the
// first member and divides by the count, and the ascent stops when sqrt(fma(dz,dz, fma(dy,dy, dx*dx))) <= 1e-3 * r (the
// OpenBLAS ddot order of np.linalg.norm) or after max_iter + 1 updates.  Every rounding is an explicit __d*_rn / __fma_rn, so
// nvcc contracts nothing.  A seed is flagged when a reduced distance lies within 2^-40 r^2 of r^2 (where scikit-learn's pow
// node bounds could decide otherwise) or a squared step within 2^-40 stop^2 of stop^2 (where another ddot order could).
#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kWarpsPerBlock = 4;
constexpr double kBand = 0x1p-40;        // flag margin, relative to r^2 and stop^2
constexpr double kPrune = 1.0 + 0x1p-30; // a node is skipped only when its lower bound^2 exceeds r^2 by this factor

struct MsArgs {
    int n, n_nodes, max_iter;
    double r, stop;
    const double* Xt;          // (n,3) points in tree order
    const long long* idx;      // (n) idx_array: tree position -> index in X
    const int* nodes;          // (n_nodes,3) idx_start, idx_end, is_leaf
    const double* bounds;      // (2,n_nodes,3) node_bounds: lower corners, then upper corners
    double* means;             // (n,3) by index in X
    int* info;                 // (n,3) by index in X: member count, iterations, flag
};

__device__ __forceinline__ double gap(double lo, double hi, double q)
{
    return fmax(fmax(__dsub_rn(lo, q), __dsub_rn(q, hi)), 0.0);
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) meanshift_kernel(MsArgs a)
{
    const int lane = threadIdx.x & 31;
    const int seed = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (seed >= a.n) return;                               // whole warps leave together
    const double r2 = __dmul_rn(a.r, a.r);
    const double r2_band = __dmul_rn(r2, kBand);
    const double r2_prune = __dmul_rn(r2, kPrune);
    const double st2 = __dmul_rn(a.stop, a.stop);
    const double st2_band = __dmul_rn(st2, kBand);
    const double* lo = a.bounds;
    const double* hi = a.bounds + 3 * (size_t)a.n_nodes;

    // the seed is X[idx[seed]] = Xt[seed]
    double qx = a.Xt[3 * (size_t)seed], qy = a.Xt[3 * (size_t)seed + 1], qz = a.Xt[3 * (size_t)seed + 2];
    int it = 0, count = 0;
    bool near = false;
    while (true) {
        double s = -0.0;                                   // lane c < 3: the chain of coordinate c; -0.0 + v == v for every v
        int m = 0;
        int node = 0;
        while (true) {
            const int* nd = a.nodes + 3 * node;
            const double g0 = gap(lo[3 * node], hi[3 * node], qx);
            const double g1 = gap(lo[3 * node + 1], hi[3 * node + 1], qy);
            const double g2 = gap(lo[3 * node + 2], hi[3 * node + 2], qz);
            const double lb2 = __dadd_rn(__dadd_rn(__dmul_rn(g0, g0), __dmul_rn(g1, g1)), __dmul_rn(g2, g2));
            const bool visit = !(lb2 > r2_prune);
            if (visit && !nd[2]) {                         // inner node: left child first
                node = 2 * node + 1;
                continue;
            }
            if (visit) {
                const int end = nd[1];
                for (int base = nd[0]; base < end; base += 32) {
                    const int p = base + lane;
                    bool in = false;
                    if (p < end) {
                        const double* x = a.Xt + 3 * (size_t)p;
                        const double dx = __dsub_rn(qx, x[0]), dy = __dsub_rn(qy, x[1]), dz = __dsub_rn(qz, x[2]);
                        const double rd = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                        in = rd <= r2;
                        near |= fabs(__dsub_rn(rd, r2)) <= r2_band;
                    }
                    unsigned members = __ballot_sync(0xffffffffu, in);
                    m += __popc(members);
                    if (lane < 3) {
                        while (members) {                  // ascending tree position
                            const int b = __ffs(members) - 1;
                            members &= members - 1;
                            s = __dadd_rn(s, a.Xt[3 * (size_t)(base + b) + lane]);
                        }
                    }
                }
            }
            while (node != 0 && (node & 1) == 0) node = (node - 1) >> 1;   // climb out of right children
            if (node == 0) break;
            ++node;                                        // left child -> its right sibling
        }
        if (m == 0) break;                                 // no point within r: the previous mean stands
        count = m;
        const double mean_c = __ddiv_rn(s, (double)m);
        const double nx = __shfl_sync(0xffffffffu, mean_c, 0);
        const double ny = __shfl_sync(0xffffffffu, mean_c, 1);
        const double nz = __shfl_sync(0xffffffffu, mean_c, 2);
        const double dx = __dsub_rn(nx, qx), dy = __dsub_rn(ny, qy), dz = __dsub_rn(nz, qz);
        const double sq = __fma_rn(dz, dz, __fma_rn(dy, dy, __dmul_rn(dx, dx)));
        near |= fabs(__dsub_rn(sq, st2)) <= st2_band;
        qx = nx; qy = ny; qz = nz;
        if (__dsqrt_rn(sq) <= a.stop || it == a.max_iter) break;
        ++it;
    }
    near = __any_sync(0xffffffffu, near);
    if (lane == 0) {
        const long long i = a.idx[seed];
        a.means[3 * i] = qx; a.means[3 * i + 1] = qy; a.means[3 * i + 2] = qz;
        a.info[3 * i] = count; a.info[3 * i + 1] = it; a.info[3 * i + 2] = near ? 1 : 0;
    }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_meanshift(int n, int n_nodes, const double* Xt, const long long* idx, const int* nodes, const double* bounds, double bandwidth,
                  double stop_thresh, int max_iter, double* means, int* info, void* stream)
{
    using namespace tgn;
    if (n < 0 || n_nodes < 1 || !(bandwidth > 0.0) || !(stop_thresh >= 0.0) || max_iter < 0) {
        set_error("meanshift: bad arguments n=%d n_nodes=%d bandwidth=%g stop_thresh=%g max_iter=%d", n, n_nodes, bandwidth, stop_thresh,
                  max_iter);
        return TGN_ERR_INVALID;
    }
    if (n == 0) return TGN_OK;
    if (!Xt || !idx || !nodes || !bounds || !means || !info) {
        set_error("meanshift: null argument");
        return TGN_ERR_INVALID;
    }
    MsArgs a;
    a.n = n; a.n_nodes = n_nodes; a.max_iter = max_iter;
    a.r = bandwidth; a.stop = stop_thresh;
    a.Xt = Xt; a.idx = idx; a.nodes = nodes; a.bounds = bounds; a.means = means; a.info = info;
    const int blocks = (n + kWarpsPerBlock - 1) / kWarpsPerBlock;
    meanshift_kernel<<<blocks, kWarpsPerBlock * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch("meanshift");
}

}  // extern "C"
