/*
 * tgn_b200.h -- C ABI of libtgn_b200.so: the H100-native (sm_90a) replacement for the native
 * layer of limhoyeon/ToothGroupNetwork's point-cloud operator hot path.
 *
 * Boundary being replaced (paths relative to /root/reference/external_libs/pointops/src):
 * the reference exposes its kernels to the pybind glue through ten `extern "C"` launchers
 * taking raw device pointers.  Part 1 below exports those ten symbols with identical
 * signatures and semantics (legacy default stream, void return, caller-owned outputs), so
 * the reference's `*_cuda.cpp` glue links against this library unchanged.  Part 2 is the
 * same operations with an explicit stream and a status code, plus the operations the
 * reference runs as PyTorch tensor code on the pointnet2 side (ball query, 3-NN, gather,
 * grouped shared-MLP set abstraction), which this library provides as fused kernels.
 *
 * Conventions: all pointers are DEVICE pointers unless stated otherwise; float = fp32,
 * int = int32; tensors are dense row-major; `stream` is a cudaStream_t passed as void*.
 * Part-2 functions return 0 on success, TGN_ERR_* otherwise (text in tgn_last_error()).
 * No function synchronises the device.  There is no CPU path.
 */
#ifndef TGN_B200_H_
#define TGN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ===================================================================================
 * Part 1 -- drop-in for the reference's extern "C" launchers.
 * =================================================================================== */

/* sampling/sampling_cuda_kernel.h:14 (definition sampling_cuda_kernel.cu:131-171).
 * b clouds packed in xyz (n_total,3) with cumulative ends offset[b]; new_offset[b] cumulative
 * sample counts; n = largest cloud size (selects the reference's block size and therefore its
 * tie-break); tmp (n_total) pre-filled by the caller (1e10), holds the running minima on
 * return; idx (m_total) receives global row ids, first sample of a cloud = its first point. */
void furthestsampling_cuda_launcher(int b, int n, const float *xyz, const int *offset,
                                    const int *new_offset, float *tmp, int *idx);

/* knnquery/knnquery_cuda_kernel.h:14 (definition knnquery_cuda_kernel.cu:111-116).
 * idx (m,nsample), dist2 (m,nsample) = squared distances, ascending; a segment with fewer
 * than nsample points leaves (segment start, 1e10) in the trailing slots. */
void knnquery_cuda_launcher(int m, int nsample, const float *xyz, const float *new_xyz,
                            const int *offset, const int *new_offset, int *idx, float *dist2);

/* grouping/grouping_cuda_kernel.h:13-14 (grouping_cuda_kernel.cu:27-41) */
void grouping_forward_cuda_launcher(int m, int nsample, int c, const float *input, const int *idx, float *output);
void grouping_backward_cuda_launcher(int m, int nsample, int c, const float *grad_output, const int *idx, float *grad_input);

/* interpolation/interpolation_cuda_kernel.h:13-14 (interpolation_cuda_kernel.cu:35-47);
 * output / grad_input are accumulated into and must be pre-zeroed by the caller. */
void interpolation_forward_cuda_launcher(int n, int c, int k, const float *input, const int *idx, const float *weight, float *output);
void interpolation_backward_cuda_launcher(int n, int c, int k, const float *grad_output, const int *idx, const float *weight, float *grad_input);

/* subtraction/subtraction_cuda_kernel.h:13-14 (subtraction_cuda_kernel.cu:32-44) */
void subtraction_forward_cuda_launcher(int n, int nsample, int c, const float *input1, const float *input2, const int *idx, float *output);
void subtraction_backward_cuda_launcher(int n, int nsample, int c, const int *idx, const float *grad_output, float *grad_input1, float *grad_input2);

/* aggregation/aggregation_cuda_kernel.h:12-17 (aggregation_cuda_kernel.cu:41-53) */
void aggregation_forward_cuda_launcher(int n, int nsample, int c, int w_c, const float *input, const float *position,
                                       const float *weight, const int *idx, float *output);
void aggregation_backward_cuda_launcher(int n, int nsample, int c, int w_c, const float *input, const float *position,
                                        const float *weight, const int *idx, const float *grad_output,
                                        float *grad_input, float *grad_position, float *grad_weight);

/* ===================================================================================
 * Part 2 -- stream-taking, status-returning entry points.
 * =================================================================================== */
#define TGN_OK 0
#define TGN_ERR_INVALID 1
#define TGN_ERR_CUDA 2

int tgn_version(void);
const char *tgn_last_error(void);          /* thread-local, valid until the next failing call */
int tgn_launch_count(void);                /* kernels launched by this library in this process */

/* FPS.  Same contract as furthestsampling_cuda_launcher; tmp may be NULL (running minima start
 * at 1e10 and are not written back) when the cloud fits the register-resident kernel.
 * `mode`: 0 = choose by b and n_max: clouds of more than 4096 points go to the bucket-pruned kernel
 *         (Morton-sorted 64-point buckets, exact; 16, 8 or 4 warps per cloud as the batch grows),
 *         smaller ones stay register-resident in one CTA / cluster;
 *         -1 = streaming kernel (needs tmp); -2 = bucket kernel, shape by batch size;
 *         -(10 + W) = bucket kernel with W in {16, 8, 4, 2, 1} warps per cloud;
 *         100*G + CS = register-resident cluster of CS CTAs (1,2,4,8) with G clouds in flight
 *         (1 or 2; G omitted = 1).  Every mode returns the same indices. */
int tgn_furthestsampling(int b, int n_max, const float *xyz, const int *offset, const int *new_offset,
                         float *tmp, int *idx, int mode, void *stream);

/* kNN.  b = number of segments (length of offset / new_offset). */
int tgn_knnquery(int b, int m, int nsample, const float *xyz, const float *new_xyz, const int *offset,
                 const int *new_offset, int *idx, float *dist2, void *stream);

/* Crop extraction: the k (<= 4096) nearest points of each of Q centres per cloud, ascending (float64 distance, index) --
 * replaces ops_utils.get_nearest_neighbor_idx (sklearn KDTree.query(k=3072) on the host, ops_utils.py:146-161).
 * xyz (B,N,3), centres (B,Q,3) -> out_idx (B,Q,k) int32, or int64 when idx64 != 0.  One CTA per centre: radix select of
 * the k-th distance, compaction, bitonic sort. */
int tgn_crop_knn(int B, int N, int Q, int k, const float *xyz, const float *centres, void *out_idx, int idx64, void *stream);

/* DBSCAN labels equal to scikit-learn's DBSCAN(eps, min_samples).fit(xyz).labels_ (float64 reduced-distance predicate, clusters
 * numbered by their smallest core index, border points take the smallest neighbouring label, noise -1): replaces the host-side
 * clustering of ops_utils.get_clustering_labels (ops_utils.py:98).  xyz (n,3) float32 DEVICE; workspace of
 * tgn_dbscan_bytes(n) DEVICE bytes; labels (n) int32, core (n) bytes (1 = core sample), n_clusters DEVICE int or NULL. */
size_t tgn_dbscan_bytes(int n);
int tgn_dbscan(int n, const float *xyz, double eps, int min_samples, void *workspace, int *labels, unsigned char *core, int *n_clusters,
               void *stream);

/* scikit-learn 1.9's KMeans(k, init="k-means++", n_init=1, algorithm="lloyd", max_iter).fit on float32 (n,3) points, one fit per
 * CTA (ops_utils.clustering_points(method="kmeans")).  B fits of points X (N,3) float32 DEVICE, fit f holding rows offsets[f] ..
 * offsets[f+1]-1 (offsets (B+1) int32 DEVICE), already centred by the host (X - X.mean(0)); 1 <= k <= 64 and k <= each fit's n.
 * Per fit, DEVICE: first (B) int32 = random_state.choice(n, p=w/w.sum()); uniforms (B, k-1, 2+int(log k)) float64 =
 * random_state.uniform draws; tol (B) float32 = mean(var(X)) * tol.  Workspace of tgn_kmeans_bytes(N, B) DEVICE bytes.
 * Outputs, DEVICE: labels (N) int32, init (B,k) int64 (the k-means++ indices), centers (B,k,3) float32 (centred), n_iter (B),
 * inertia (B) float32, relocated (B) int32 = 1 when a cluster emptied (scikit-learn relocates it; not restated, the other
 * outputs of that fit are then meaningless). */
size_t tgn_kmeans_bytes(long long n_total, int B);
int tgn_kmeans(int B, long long n_total, int k, int max_iter, const int *offsets, const float *X, const int *first, const double *uniforms,
               const float *tol, void *workspace, int *labels, long long *init, float *centers, int *n_iter, float *inertia, int *relocated,
               void *stream);

/* The seed ascent of scikit-learn 1.9's MeanShift(bandwidth, max_iter).fit on float64 (n,3) points with seeds = X: each
 * seed's _mean_shift_single_seed, one warp per seed (the elongated-cluster split of ops_utils.get_clustering_labels).  The
 * KD tree is scikit-learn's KDTree(X, leaf_size=30).get_arrays(), DEVICE: Xt (n,3) float64 = X[idx_array]; idx (n) int64 =
 * idx_array; nodes (n_nodes,3) int32 = idx_start, idx_end, is_leaf; bounds (2,n_nodes,3) float64 = node_bounds.
 * stop_thresh = 1e-3 * bandwidth as the host computes it.  Outputs by index in X, DEVICE: means (n,3) float64 (the seed's
 * final mean), info (n,3) int32 = member count of the last query (0 when it found no point), completed iterations, and a flag
 * (1 when a reduced distance came within 2^-40 r^2 of r^2 or a squared step within 2^-40 stop^2 of stop^2: only such a seed
 * may differ from scikit-learn, and the host redoes it). */
int tgn_meanshift(int n, int n_nodes, const double *Xt, const long long *idx, const int *nodes, const double *bounds, double bandwidth,
                  double stop_thresh, int max_iter, double *means, int *info, void *stream);

/* scikit-learn 1.9's KDTree(xyz, leaf_size) built on the device, bit for bit: the arrays of KDTree.get_arrays() for float64
 * (n,3) points (the label transfers' tie fallback, MeanShift's tree).  tgn_kdtree_nodes(n, leaf_size) = n_nodes
 * (2^n_levels - 1, -1 for arguments out of range); a DEVICE workspace of tgn_kdtree_bytes(n, leaf_size) bytes.  Outputs,
 * DEVICE: idx_array (n) int64; node_data (n_nodes) records of scikit-learn's NodeData_t {idx_start, idx_end, is_leaf int64;
 * radius float64}, the radius left NaN; node_bounds (2, n_nodes, 3) float64.  No host synchronisation.  1 <= n <= 2^30,
 * finite coordinates (not checked here), leaf_size >= 1.  tgn_kdtree_radius fills the radius of HOST copies of node_data from
 * node_bounds the way scikit-learn's init_node computes it, with the C library's pow. */
int tgn_kdtree_nodes(int n, int leaf_size);
size_t tgn_kdtree_bytes(int n, int leaf_size);
int tgn_kdtree_build(int n, int leaf_size, const double *xyz, long long *idx_array, long long *node_data, double *node_bounds,
                     void *workspace, void *stream);
void tgn_kdtree_radius(int n_nodes, const double *node_bounds, double *node_data);

/* scikit-learn 1.9's KDTree.query(queries, k) (single tree, depth first, sorted results) over the arrays tgn_kdtree_build
 * writes, one warp per row.  xyz (n,3) float64 in original order, idx_array (n) int64, node_data (n_nodes,4) int64 (the radius
 * is not read), node_bounds (2,n_nodes,3) float64, queries (m,3) float64 finite, all DEVICE.  rows (n_rows) int64 DEVICE row
 * numbers, or NULL for every row; only the listed rows of the outputs are written (a number outside [0, m) is skipped).
 * Outputs, DEVICE: idx (m,k) int64; dist (m,k) float64 = sqrt of the reduced distance, optional (NULL); flag (m) bytes: 1 when a
 * trim or child-order decision compared a node bound whose squares were not all exact within a relative 2^-40 (only there may
 * scikit-learn's pow decide otherwise); a row with flag 0 is scikit-learn's answer, indices and distance bits.  1 <= n <= 2^30,
 * n_nodes = 2^L - 1 with 2^(L-1) <= n, 1 <= k <= min(n, 63). */
int tgn_kdtree_query(int n, int n_nodes, int k, const double *xyz, const long long *idx_array, const long long *node_data,
                     const double *node_bounds, int m, const double *queries, const long long *rows, int n_rows, long long *idx,
                     double *dist, unsigned char *flag, void *stream);

/* Exact float64 kNN with a fused label vote: the answer of sklearn KDTree(xyz).query(queries, k) -- boundary detection of
 * InferencePipeLine.get_boundary_sampled_feats (inference_pipeline_tgn.py:289-330).  xyz (n,3) and queries (m,3) float64
 * DEVICE; 1 <= k <= 64, k <= n.  Distances d2 = (dx*dx + dy*dy) + dz*dz in float64 without contraction, neighbours ascending
 * by (d2, index).  Each call builds a uniform grid into a DEVICE workspace of tgn_knn_f64_bytes(n) bytes and queries it.
 * Outputs, each optional (NULL): idx (m,k) int64; dist (m,k) float64 = correctly rounded sqrt(d2); nn0 (m) int32 = index of
 * the nearest point; agree (m) int32 = how many of the k neighbours carry labels[nn0] (needs labels (n) int32). */
size_t tgn_knn_f64_bytes(int n);
int tgn_knn_f64(int n, int m, int k, const double *xyz, const double *queries, void *workspace, const int *labels, long long *idx,
                double *dist, int *nn0, int *agree, void *stream);

/* The same kNN with the grid built once and queried many times (KDTree(X) once, .query(...) per query set): tgn_knn_f64_build
 * writes the grid of xyz (n,3) float64 DEVICE into a caller-owned DEVICE workspace of tgn_knn_f64_bytes(n) bytes;
 * tgn_knn_f64_query answers queries (m,3) against it without writing to it (xyz and n are those of the build; any number of
 * queries may share one built workspace).  tgn_knn_f64 is build + query.  Outputs as above, plus tie (m) bytes, optional:
 * tie[i] = 1 exactly when two adjacent keys among query i's min(k+1, n) smallest (d2, index) have equal d2, else 0.  A row with
 * tie[i] = 0 has one answer under every tie-break rule (sklearn's KDTree returns exactly it).  With tie, 1 <= k <= 63. */
int tgn_knn_f64_build(int n, const double *xyz, void *workspace, void *stream);
int tgn_knn_f64_query(int n, int m, int k, const double *xyz, const double *queries, const void *workspace, const int *labels,
                      long long *idx, double *dist, int *nn0, int *agree, unsigned char *tie, void *stream);

/* Exact feature-space kNN of DGCNN (models/modules/dgcnn.py:4-10): per cloud, the k largest of
 * v_ij = fl(fl(-xx_j - fl(-2*dot_ij)) - xx_i), dot_ij = the in-order FFMA chain over c, with the indices and values
 * pairwise_distance.topk(k, dim=-1) returns, without the N x N matrix.  x (b, c, n) float32 DEVICE, element (bi, ci, ni) at
 * x[bi*stride_b + ci*stride_c + ni*stride_n]; xx (b, n) float32 DEVICE = torch.sum(x**2, dim=1) as the caller computed it;
 * 1 <= c <= 64, 1 <= k <= 32, n >= k.  Outputs idx (b, n, k) int64 and val (b, n, k) float32 (optional, NULL), in topk's
 * sorted order (a NaN value is returned as the canonical NaN). */
int tgn_knn_feat(int b, int n, int c, int k, const float *x, long long stride_b, long long stride_c, long long stride_n,
                 const float *xx, long long *idx, float *val, void *stream);

/* kNN through a per-segment uniform grid: identical answers to tgn_knnquery (distinct distances: order-independent;
 * ties among the k+1 best: the query is re-run with the reference's index-order heap), ~100x fewer distance evaluations
 * on 24k-point clouds.  The grid depends only on (xyz, offset): build it once into a caller-owned DEVICE workspace of
 * tgn_knn_grid_bytes(b, n_total) bytes and reuse it for every query set / k against that point set. */
size_t tgn_knn_grid_bytes(int b, int n_total);
int tgn_knn_grid_build(int b, int n_total, const float *xyz, const int *offset, void *workspace, void *stream);
int tgn_knn_grid_query(int b, int n_total, int m, int nsample, const float *xyz, const float *new_xyz, const int *offset,
                       const int *new_offset, const void *workspace, int *idx, float *dist2, void *stream);

int tgn_grouping_forward(int m, int nsample, int c, const float *input, const int *idx, float *output, void *stream);
int tgn_grouping_backward(int m, int nsample, int c, const float *grad_output, const int *idx, float *grad_input, void *stream);
int tgn_interpolation_forward(int n, int c, int k, const float *input, const int *idx, const float *weight, float *output, void *stream);
int tgn_interpolation_backward(int n, int c, int k, const float *grad_output, const int *idx, const float *weight, float *grad_input, void *stream);
/* output[n,:] += sum_i input[idx[n,i],:] * weight[n,i].  fused = 1: the FMA chain of interpolation_cuda_kernel.cu:5-18
 * (== tgn_interpolation_forward); fused = 0: product rounded, then added -- the arithmetic of the torch loop in
 * pointops.interpolation (pointops.py:177-179), which is what the models call. */
int tgn_weighted_gather(int n, int c, int k, const float *input, const int *idx, const float *weight, float *output, int fused, void *stream);
/* Deterministic, ORDER-EXACT scatter-add backwards.  The reference's live callers gather with torch advanced indexing,
 * whose backward (index_put_ accumulate) adds every destination row's contributions sequentially in ascending source
 * position.  tgn_csr_build inverts an index tensor once (keys[M] -> per destination row the ascending list of source
 * positions) into a DEVICE workspace of tgn_csr_bytes(M, n_rows); the two backwards below then reproduce torch's sums
 * bit for bit, without value atomics.
 *   tgn_gather_backward_det:           grad_in[r,:] = sum_{p : keys[p]=r, ascending} grad_out[p,:]      (grad_out (M,c))
 *   tgn_weighted_gather_backward_det:  keys = idx (n,k) flattened; grad_out (n,c), weight (n,k):
 *        per i: G_i[r,:] = sum_{n ascending, idx[n,i]=r} grad_out[n,:]*weight[n,i];  grad_in = ((G_{k-1}+G_{k-2})+...)+G_0
 *        -- the order in which autograd sums the k index_put results of pointops.interpolation (pointops.py:177-179);
 *        single != 0: one accumulation over all (n,i) in ascending n*k+i -- the backward of pointnet2_utils.py:340.
 *   c == 1 follows torch's kernel for one-element slices: for a row (of each accumulation) with d terms, lane L of a warp adds
 *        terms L, 32+L, ... below F = 32*floor(d/32), the 32 lane sums are reduced by shfl_down (16, 8, 4, 2, 1), then terms
 *        F .. d-1 are added in order (d < 32: the plain ascending sum).  Every c > 1 is the ascending sequential sum.
 *   Keys outside [0, n_rows) are dropped (they add to no row); a row without keys gets 0.  M == 0 is valid: tgn_csr_build writes
 *        an empty inverse (row_start all zero) and both backwards then write zeros.  k > 8 is refused (callers use atomics). */
size_t tgn_csr_bytes(long long M, int n_rows);
int tgn_csr_build(long long M, int n_rows, const int *keys, void *workspace, void *stream);
int tgn_gather_backward_det(long long M, int n_rows, int c, const void *workspace, const float *grad_out, float *grad_in, void *stream);
int tgn_weighted_gather_backward_det(long long M, int n_rows, int c, int k, int single, const void *workspace, const float *grad_out,
                                     const float *weight, float *grad_in, void *stream);

int tgn_subtraction_forward(int n, int nsample, int c, const float *input1, const float *input2, const int *idx, float *output, void *stream);
int tgn_subtraction_backward(int n, int nsample, int c, const int *idx, const float *grad_output, float *grad_input1, float *grad_input2, void *stream);
int tgn_aggregation_forward(int n, int nsample, int c, int w_c, const float *input, const float *position, const float *weight,
                            const int *idx, float *output, void *stream);
int tgn_aggregation_backward(int n, int nsample, int c, int w_c, const float *input, const float *position, const float *weight,
                             const int *idx, const float *grad_output, float *grad_input, float *grad_position,
                             float *grad_weight, void *stream);

/* Ball query: pointnet2_utils.query_ball_point (external_libs/pointnet2_utils/pointnet2_utils.py:120-144).
 * xyz (B,N,3), new_xyz (B,S,3) -> group_idx (B,S,nsample): the first nsample point indices in
 * ascending order whose EXPANDED squared distance (-2ab + |a|^2 + |b|^2, evaluated in the
 * reference's rounding order) is not > r2, padded with the first hit; N in every slot when the
 * ball is empty.  r2 must be float32(radius**2).  idx64 is a bit set: bit 0 writes int64 (the
 * reference's dtype) instead of int32; by default clouds of >= 8192 points whose balls are sparse
 * are answered by a uniform-grid kernel and the rest by an index-order tile scan (same result);
 * bit 2 (4) forces the tile scan, bit 3 (8) the grid, bit 1 (2) a streaming scan (experiments).
 * Bits 4 (16) / 5 (32): |new_xyz|^2 / |xyz|^2 rounded as (x*x + z*z) + y*y instead of (x*x + y*y) + z*z --
 * torch.sum(p ** 2, -1) on CUDA takes the first form for a contiguous (..., 3) operand and the second for a strided
 * view (and always on the CPU); the Python layer sets the bits from the layout the reference's call would see. */
int tgn_ball_query(int B, int N, int S, float r2, int nsample, const float *xyz, const float *new_xyz,
                   void *group_idx, int idx64, void *stream);

/* 3 nearest coarse points by the same expanded distance (pointnet2_utils.py:333-335):
 * xyz1 (B,N,3) fine, xyz2 (B,S,3) coarse, S >= 3 -> dist (B,N,3) ascending, idx (B,N,3) int32. */
int tgn_three_nn(int B, int N, int S, const float *xyz1, const float *xyz2, float *dist, int *idx, void *stream);
/* Same with `order`: bit 0 / bit 1 = |xyz1|^2 / |xyz2|^2 in the contiguous-reduce rounding (see tgn_ball_query). */
int tgn_three_nn_ex(int B, int N, int S, const float *xyz1, const float *xyz2, float *dist, int *idx, int order, void *stream);

/* The matrix itself (pointnet2_utils.square_distance :20-41): src (B,N,3), dst (B,M,3) -> out (B,N,M), expanded form, `order` as in
 * tgn_three_nn_ex (bit 0: src, bit 1: dst).  Forward only; the Python wrapper keeps torch's formulation under autograd. */
int tgn_square_distance(int B, int N, int M, const float *src, const float *dst, float *out, int order, void *stream);

/* Weighted 3-point interpolation (pointnet2_utils.py:337-340): weights 1/(dist+1e-8) normalised,
 * points2 (B,S,C) point-major -> out (B,N,C). */
int tgn_three_interpolate(int B, int N, int S, int C, const float *points2, const float *dist, const int *idx,
                          float *out, void *stream);
/* norm_alt != 0: the normaliser is summed as (r0 + r2) + r1, torch's CUDA reduce order for the contiguous (B,N,3)
 * reciprocal tensor; 0: (r0 + r1) + r2, the CPU order. */
int tgn_three_interpolate_ex(int B, int N, int S, int C, const float *points2, const float *dist, const int *idx,
                             float *out, int norm_alt, void *stream);

/* Batched row gather: pointnet2_utils.index_points (pointnet2_utils.py:44-61).
 * points (B,N,C), idx (B,M) int32 -> out (B,M,C). */
int tgn_gather_rows(int B, int N, int M, int C, const float *points, const int *idx, float *out, void *stream);

/* (B,C,N) -> (B,N,C) and back (the reference permutes with torch; here one tiled kernel). */
int tgn_transpose_cn(int B, int C, int N, const float *in, float *out, void *stream);

/* Fused set-abstraction body: gather -> [xyz_rel | feats] -> L x (1x1 conv + bias + ReLU) -> max
 * over the K neighbours, without materialising the grouped tensor
 * (PointNetSetAbstraction.forward pointnet2_utils.py:213-239 / Msg :261-299, eval-mode BatchNorm
 * folded into weight/bias by the caller).
 *   xyz (B,N,3); feats (B,N,D) point-major or NULL (D = 0); new_xyz (B,S,3); group_idx (B,S,K) int32
 *   xyz_first: 1 -> channels [xyz_rel, feats] (SSG, :169), 0 -> [feats, xyz_rel] (MSG, :285)
 *   a group_idx entry outside [0, N) (the ball query's N for an empty ball) is an all-zero operand row
 *   n_layers in [1,4]; channels[n_layers+1] HOST array, channels[0] = 3 + D; every width <= 128
 *   weights[l] (C_{l+1}, C_l) row-major DEVICE, biases[l] (C_{l+1}) DEVICE; the two pointer arrays are HOST arrays
 *   out: channel-first (B, out_c_total, S); this branch writes channels [out_c_offset, +C_last)
 *   engine: 0 = auto (2 when the shape fits it, else 3, else 1), 1 = fp32 CUDA-core kernel (exact FMA),
 *           2 = tensor-core (wgmma) 3xTF32 kernel (widths <= 64, any K <= 128, ~2^-21; operands and weights within 220 KB of
 *           shared memory: four 64-wide layers are refused), 3 = tensor-core kernel for wide layers
 *           (first layer 3xTF32, later layers as three bf16x2-split MMAs, ~1e-5; at least two layers, K in {16,32,64,128},
 *           within 224 KB of shared memory: three 128-wide layers are refused),
 *           5 = engine 2 in half-size CTAs.  Any other value is refused (engine 4 was Blackwell-only and is gone). */
int tgn_sa_group_mlp_max(int B, int N, int S, int K, int D, const float *xyz, const float *feats, const float *new_xyz,
                         const int *group_idx, int xyz_first, int n_layers, const int *channels,
                         const float *const *weights, const float *const *biases, float *out, int out_c_total,
                         int out_c_offset, int engine, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * 1x1-convolution chains with BATCH-STATISTICS BatchNorm (any width), one launch per layer
 * (PointNetSetAbstraction(Msg).forward pointnet2_utils.py:232-237 / :289-294 and
 * PointNetFeaturePropagation.forward :346-352 with BatchNorm in training mode -- which is how every
 * reference call site, inference included, runs them -- and in eval mode for widths the single-kernel
 * engines above do not take).  Layer l computes the RAW pre-activation, channel-major:
 *      y[c, r] = sum_k W[c, k] * act(x)[r, k] + bias[c],   r in [0, rows)
 * where act() is the previous layer's BatchNorm + ReLU applied while the operand is built
 * (in_affine: 0 none, 1 from the fp64 batch sums `in_stats` = {sum[cin], sumsq[cin]} over `rows` rows,
 * 2 from running statistics).  wgmma, operands split into three bf16 parts (six MMAs per K step, fp32-grade:
 * batch-statistics BatchNorm amplifies rounding differences) or two (`precision` = 2: three MMAs, ~1e-5).
 * mode 0: the operand row r = (b, n), b = r / rows_per_batch, is read from up to two strided segments,
 *         x[k] = seg_ptr[i][b*seg_batch_stride[i] + n*seg_row_stride[i] + k'*seg_chan_stride[i]] (strides in floats);
 * mode 1: neighbourhood gather, r = ((b*S + s)*K + j): [feats[b, gidx[r], :] | xyz[b, gidx[r]] - new_xyz[b, s]]
 *         (xyz_first = 0, MSG order :285) or [xyz - centre | feats] (xyz_first = 1, SSG order :169); cin = D + 3.
 * mode 2: DGCNN edge feature (get_graph_feature, models/modules/dgcnn.py:13-41), r = ((b*N + n)*K + j), m = gidx[r] in [0, N):
 *         [x[b, :, m] - x[b, :, n] | x[b, :, n]] with x = edge_x read through edge_stride = its (b, c, n) strides in floats;
 *         cin = 2 * edge_C, rows a multiple of N * K.  A row whose m is out of range is a zero row.
 * in_act: the activation applied after the input BatchNorm: 0 = ReLU, 1 = LeakyReLU (v > 0 ? v : v * in_act_slope).
 * cloud_bias (optional, (B, cout)): y[c, r] += cloud_bias[r / rows_per_batch, c] after the bias -- an operand segment that is
 * constant over each cloud's rows, added once in fp32 instead of through the MMAs (tgn_pw_cloud_bias computes it).
 * Outputs, each optional: y (cout, rows); stats (2*cout doubles, ACCUMULATED: caller zeroes) = per-channel
 * sum / sum of squares of y; ymax / ymin (cout, rows/group) = extrema over groups of `group` consecutive rows
 * (the max over the K neighbours must wait for the BatchNorm scale's sign, so both are kept); with
 * extrema_atomic != 0 they are merged with atomics into buffers the caller pre-filled with -inf / +inf
 * (required when 128 % group != 0; when 64 % group != 0 with accum = 1).  w_packed: tgn_pw_pack_weights of the (cout, cin) weight.
 * accum = 1: promoted accumulation -- 128-row tiles whose tensor-core accumulator is added into an fp32 register total with a
 * round-to-nearest add every K step (16 values of K) and restarted, so the accumulators' truncation is confined to one
 * chunk; for layers followed by BatchNorm on running statistics, which does not subtract that truncation again.  The field sits
 * in what was padding: an all-zero descriptor launches exactly what it did before the field existed.
 * in_update_running != 0 with in_affine == 1 applies torch's momentum update to in_running_mean / _var once. */
typedef struct {
    int rows, rows_per_batch, cin, cout;
    int mode;
    int accum;              /* 0: one tensor-core accumulator over all of K; 1: promoted (see above) */
    const float *seg_ptr[2];
    int seg_channels[2];
    long long seg_batch_stride[2], seg_row_stride[2], seg_chan_stride[2];
    const float *xyz, *feats, *new_xyz;
    const int *gidx;
    int N, S, K, D, xyz_first;
    int in_affine, in_update_running;
    const double *in_stats;
    const float *in_gamma, *in_beta;
    float *in_running_mean, *in_running_var;
    float in_eps, in_momentum;
    const void *w_packed;
    const float *bias;
    float *y;
    double *stats;
    float *ymax, *ymin;
    int group, extrema_atomic;
    int precision;          /* 0 / 3: three bf16 parts per operand, six MMAs per K step (fp32-grade); 2: two parts, three MMAs (~1e-5) */
    const float *edge_x;    /* mode 2 */
    long long edge_stride[3];
    int edge_C;
    int in_act;
    float in_act_slope;
    const float *cloud_bias;
} tgn_pw_layer_t;

/* Final BatchNorm (+ activation) of a chain into a channel-first tensor:
 *   out[b, out_c_offset + c, n] = act(scale_c * v + shift_c),  v = src[c, b*rows_per_batch + n]
 * or, when ymin != NULL, v = (scale_c >= 0 ? src : ymin)[c, ...] (src = the max).  `affine` as in_affine above
 * (0 = identity), statistics over stat_rows rows.  act: LeakyReLU (v > 0 ? v : v * act_slope) when act == 1, else ReLU
 * when relu != 0, else none. */
typedef struct {
    int rows, rows_per_batch, channels, out_channels, out_c_offset, relu;
    const float *src, *ymin;
    float *out;
    int affine, update_running;
    const double *stats;
    long long stat_rows;
    const float *gamma, *beta;
    float *running_mean, *running_var;
    float eps, momentum;
    int act;
    float act_slope;
} tgn_pw_apply_t;

/* Fused forward of blocks.PointTransformerLayer (models/modules/cbl_point_transformer/blocks.py:14-44; SURVEY 8(f)-3): vector
 * self-attention over the K neighbours idx[i, :] of every point, share_planes = 8, in up to four passes over the gathers (one per
 * BatchNorm that runs on batch statistics + the output pass); nothing of size (n, K, c) is materialised.
 *   p (n,3); xq, xk, xv (n,c) = linear_q/k/v(x) (left to the caller's GEMMs); idx (n,K) int32 (kNN of p in p); out (n,c)
 *   linear_p = Linear(3,3) [p_w0 (3,3), p_b0] -> BatchNorm1d(3) [p_*] -> ReLU -> Linear(3,c) [p_w1 (c,3), p_b1]
 *   linear_w = BatchNorm1d(c) [a_gamma..] -> ReLU -> Linear(c, c/8) [a_w (c/8,c), a_b] -> BatchNorm1d(c/8) [b_gamma..] -> ReLU
 *              -> Linear(c/8, c/8) [b_w, b_b]
 *   bn_mode[i]: 1 = batch statistics (stats_* = zeroed fp64 {sum[ch], sumsq[ch]} scratch, filled by the passes), 2 = running
 *   statistics; update_running != 0 applies torch's momentum update to the *_rmean / *_rvar of the BatchNorms in mode 1.
 *   The passes ADD into stats_*: the caller zeroes them before every launch.
 *   idx entries must lie in [0, n); they are not checked.
 * c in {16, 32, 64, 128, 256, 512}, K <= 64; c = 16 runs two queries per warp, one per half-warp. */
typedef struct {
    int n, c, K;
    const float *p, *xq, *xk, *xv;
    const int *idx;
    float *out;
    const float *p_w0, *p_b0, *p_w1, *p_b1;
    const float *p_gamma, *p_beta; float *p_rmean, *p_rvar; float p_eps, p_momentum;
    const float *a_gamma, *a_beta; float *a_rmean, *a_rvar; float a_eps, a_momentum;
    const float *a_w, *a_b;
    const float *b_gamma, *b_beta; float *b_rmean, *b_rvar; float b_eps, b_momentum;
    const float *b_w, *b_b;
    double *stats_p, *stats_a, *stats_b;
    int bn_mode[3];
    int update_running;
} tgn_pt_layer_t;
int tgn_pt_layer_forward(const tgn_pt_layer_t *layer, void *stream);
int tgn_pt_layer_struct_size(void);
/* layers with fewer queries than this run one CTA per query instead of one warp per query (default 1024); returns the old value.
 * c = 16 layers always run two queries per warp: the threshold does not apply to them. */
int tgn_pt_layer_set_cta_threshold(int n_queries);
/* the current threshold, unchanged */
int tgn_pt_layer_cta_threshold(void);
/* The same launch with the fp64 batch sums of its output, for the BatchNorm that follows the layer in PointTransformerBlock
 * (blocks.py:131, bn2): out_stats (2c doubles, ACCUMULATED: caller zeroes) = {sum[ch], sumsq[ch]} of out over its n rows, each
 * element added to the fp64 sums as it is written.  `layer` is exactly what tgn_pt_layer_forward takes, and out is bit for bit
 * what that call writes. */
typedef struct {
    tgn_pt_layer_t layer;
    double *out_stats;
} tgn_pt_layer_sums_t;
int tgn_pt_layer_forward_sums(const tgn_pt_layer_sums_t *p, void *stream);
int tgn_pt_layer_sums_struct_size(void);

size_t tgn_pw_packed_bytes(int cout, int cin);
int tgn_pw_struct_size(int which);         /* sizeof(tgn_pw_layer_t) (0) / sizeof(tgn_pw_apply_t) (1): binding self-check */
int tgn_pw_pack_weights(int cout, int cin, const float *w, void *packed, void *stream);
int tgn_pw_layer_forward(const tgn_pw_layer_t *layer, void *stream);
int tgn_pw_apply(const tgn_pw_apply_t *p, void *stream);
int tgn_pw_fill(float *ptr, long long n, float value, void *stream);
/* out[b*cout + c] = sum_k w[c*w_row_stride + k] * g[b*g_batch_stride + k], k < cin, accumulated in fp64 and rounded once */
int tgn_pw_cloud_bias(int B, int cout, int cin, const float *w, long long w_row_stride, const float *g, long long g_batch_stride,
                      float *out, void *stream);
/* The point-transformer decoder's final BatchNorm with TransitionUp's interpolated addend (pt_head.cu; blocks.py:109-110):
 *   out[r, c] = act(scale_c * src[c, r] + shift_c) + (((0 + f[i0, c] * w0) + f[i1, c] * w1) + f[i2, c] * w2),
 *   (i_j, w_j) = (idx[3 r + j], w[3 r + j]), every product and sum rounded on its own: pointops.interpolation's torch loop
 *   followed by the add, in torch's order.  `apply` carries rows, channels, src (channels, rows), the BatchNorm (affine,
 *   stats, stat_rows, gamma ... momentum, update_running) and the activation (relu / act) exactly as for tgn_pw_apply; its
 *   rows_per_batch, out_channels and out_c_offset are not used, ymin must be NULL, and out is (rows, channels) ROW-MAJOR.
 *   f == NULL: no addend (a row-major tgn_pw_apply).  f is (f_rows, channels) row-major; idx entries must lie in [0, f_rows). */
typedef struct {
    tgn_pw_apply_t apply;
    const float *f;
    const int *idx;
    const float *w;
    int f_rows;
} tgn_pt_up_apply_t;
int tgn_pt_up_apply(const tgn_pt_up_apply_t *p, void *stream);

/* PointTransformerBlock's last BatchNorm, residual and ReLU (pt_block.cu; blocks.py:132-134):
 *   out[r, c] = relu(fl(bn3(src[c, r])) + identity[r, c])
 * the BatchNorm value rounded to fp32 first (subtract-first, as tgn_pw_apply), then one fp32 add, then the ReLU -- torch's
 * bn3(...) followed by the in-place += and relu.  `apply` carries rows, channels, src (channels, rows) and the BatchNorm exactly as
 * for tgn_pw_apply; relu != 0 applies the ReLU after the add; rows_per_batch, out_channels and out_c_offset are not used, ymin must
 * be NULL and act 0, and out is (rows, channels) ROW-MAJOR.  identity is (rows, channels) row-major with row stride
 * identity_row_stride (in floats); it is only read and must not overlap out. */
typedef struct {
    tgn_pw_apply_t apply;
    const float *identity;
    long long identity_row_stride;
} tgn_pt_res_apply_t;
int tgn_pt_res_apply(const tgn_pt_res_apply_t *p, void *stream);
int tgn_pt_res_apply_struct_size(void);    /* sizeof(tgn_pt_res_apply_t): binding self-check */

/* MultiHead's concat-and-classify (heads.py:53-60 with combine = concat) without the upsampled copies:
 *   out[r, j] = b[j] + sum_s sum_{c<32} W[j, 32 s + c] * lat_s[c, nn_s[r]],   r < n0, j < k
 * lat_s: level s's latent, (32, n[s]) channel-major; nn_s: (n0) int32, the k = 1 neighbour of each level-0 point in level s,
 * or NULL for the identity (n[s] == n0).  W (k, 32 levels) row-major, b (k) or NULL; out (n0, k) row-major.  fp32 FFMA from
 * +0 in increasing column order, then + b[j].  1 <= levels <= 8, 1 <= k <= 32; nn entries must lie in [0, n[s]). */
#define TGN_HEAD_MAX_LEVELS 8
typedef struct {
    int n0, k, levels;
    const float *lat[TGN_HEAD_MAX_LEVELS];
    const int *nn[TGN_HEAD_MAX_LEVELS];
    int n[TGN_HEAD_MAX_LEVELS];
    const float *w, *b;
    float *out;
} tgn_head_classify_t;
int tgn_head_classify(const tgn_head_classify_t *p, void *stream);
int tgn_pt_head_struct_size(int which);    /* sizeof(tgn_pt_up_apply_t) (0) / sizeof(tgn_head_classify_t) (1): binding self-check */

/* PointNet's per-cloud transforms (pw_transform.cu): out[b, j, n] = sum_{i < ct} x[b, i, n] * t[b*t_batch_stride + i*ct + j] for
 * j < ct (fp32 FFMA from +0 in increasing i), and out[b, ct + c, n] = x[b, ct + c, n] bit for bit for c < cpass.  x and out are
 * addressed through (batch, channel, point) element strides and must not overlap.  1 <= ct <= 128. */
int tgn_pw_cloud_transform(int B, int N, int ct, int cpass, const float *x, long long xs_b, long long xs_c, long long xs_n,
                           const float *t, long long t_batch_stride, float *out, long long os_b, long long os_c, long long os_n,
                           void *stream);

#ifdef __cplusplus
}
#endif
#endif /* TGN_B200_H_ */
