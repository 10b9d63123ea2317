"""oracle/scatter.py -- restatement of one launch of the gather family and its scatter-add backwards (TEST INFRASTRUCTURE ONLY).

Every backward here is a scatter-add: element (r, ch) of the result sums the terms of the source positions p whose key is r.
For each element this module returns

* ``f64``: the sum of its terms in float64 (products of float32 operands formed exactly in float64);
* ``mag``: the magnitude ``sum |t_i|`` of the same terms;
* ``d``: the number of terms;
* ``f32`` (order-exact backwards only): the float32 sum in the order torch's ``index_put_(accumulate=True)`` takes on CUDA.

torch adds a destination row's contributions sequentially in ascending source position, except for slices of ONE element
(c == 1), which its ``indexing_backward_kernel_stride_1`` sums in a warp: lane L adds t_L, t_(32+L), ... below
F = 32 * floor(d / 32), the 32 lane sums are reduced by shfl_down (offsets 16, 8, 4, 2, 1), and lane 0 adds t_F .. t_(d-1)
after that (d < 32 is the plain sequential sum).  ``order="seq"`` is the sequential sum for every c, as torch's CPU
``index_add_`` takes it.

Keys outside [0, n_rows) are dropped: they contribute to no row.  A row without keys sums to zero.  ``bound`` is the
element-wise tolerance ``(d + 1) * 2**-24 * mag`` of a float32 evaluation that sums the float32-rounded terms in any order.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np

U32 = 2.0 ** -24


class Scatter(NamedTuple):
    f64: np.ndarray
    mag: np.ndarray
    d: np.ndarray
    f32: Optional[np.ndarray] = None


def bound(s: Scatter) -> np.ndarray:
    return (s.d + 1) * U32 * s.mag


def inverse(keys, n_rows: int):
    """(row_start (n_rows + 1), order): the in-range source positions by key, ascending inside each row (a stable argsort)."""
    keys = np.asarray(keys).reshape(-1).astype(np.int64)
    pos = np.nonzero((keys >= 0) & (keys < n_rows))[0]
    order = pos[np.argsort(keys[pos], kind="stable")]
    row_start = np.zeros(n_rows + 1, np.int64)
    np.cumsum(np.bincount(keys[pos], minlength=n_rows), out=row_start[1:])
    return row_start, order


def _seq_f32(terms: np.ndarray, row_start: np.ndarray) -> np.ndarray:
    """Per row, ((0 + t_0) + t_1) + ... in float32; terms (M', c) in CSR order."""
    n = row_start.shape[0] - 1
    d = np.diff(row_start)
    acc = np.zeros((n, terms.shape[1]), np.float32)
    by = np.argsort(-d, kind="stable")
    ds = d[by]
    for j in range(int(d.max()) if n else 0):
        act = by[:int(np.count_nonzero(ds > j))]
        acc[act] += terms[row_start[act] + j]
    return acc


def _stride1_f32(terms: np.ndarray, row_start: np.ndarray) -> np.ndarray:
    """Per row, the order of torch's indexing_backward_kernel_stride_1 (see the module docstring), column by column."""
    n = row_start.shape[0] - 1
    d = np.diff(row_start)
    c = terms.shape[1]
    lanes = np.zeros((n, 32, c), np.float32)
    passes = d // 32
    ar = np.arange(32)
    for i in range(int(passes.max()) if n else 0):
        act = np.nonzero(passes > i)[0]
        lanes[act] += terms[row_start[act, None] + 32 * i + ar]
    off = 16
    while off:
        lanes[:, :off] = lanes[:, :off] + lanes[:, off:2 * off]
        off //= 2
    g = lanes[:, 0].copy()
    full = passes * 32
    tail = d - full
    for j in range(int(tail.max()) if n else 0):
        act = np.nonzero(tail > j)[0]
        g[act] += terms[row_start[act] + full[act] + j]
    return np.float32(0.0) + g


def index_put_f32(terms, keys, n_rows: int, order: str = "cuda") -> np.ndarray:
    """zeros((n_rows, c)).index_put_((keys,), terms, accumulate=True) in float32, in torch's order: "cuda" (stride_1 order
    when c == 1, else sequential), "seq" (sequential, torch on the CPU) or "rev" (sequential in DESCENDING position)."""
    terms = np.asarray(terms, np.float32)
    keys = np.asarray(keys).reshape(-1)
    terms = terms.reshape(keys.shape[0], terms.shape[-1])
    if order == "rev":
        terms, keys = terms[::-1], keys[::-1]
    row_start, order_ = inverse(keys, n_rows)
    t = terms[order_]
    if order == "cuda" and terms.shape[1] == 1:
        return _stride1_f32(t, row_start)
    return _seq_f32(t, row_start)


def _scatter64(keys, terms64: np.ndarray, n_rows: int):
    """float64 sums, magnitudes and term counts of terms (M, c) scattered by keys (M,) into (n_rows, c)."""
    keys = np.asarray(keys).reshape(-1).astype(np.int64)
    terms64 = terms64.reshape(keys.shape[0], terms64.shape[-1])
    c = terms64.shape[1]
    ok = (keys >= 0) & (keys < n_rows)
    k, t = keys[ok], terms64[ok]
    flat = (k[:, None] * c + np.arange(c)).reshape(-1)
    f64 = np.bincount(flat, weights=t.reshape(-1), minlength=n_rows * c).reshape(n_rows, c)
    mag = np.bincount(flat, weights=np.abs(t).reshape(-1), minlength=n_rows * c).reshape(n_rows, c)
    d = np.broadcast_to(np.bincount(k, minlength=n_rows)[:, None], (n_rows, c))
    return f64, mag, d


# ------------------------------------------------------------------------------------------------------------- backwards
def gather_backward(grad_out, keys, n_rows: int, order: str = "cuda") -> Scatter:
    """grad wrt x of x[keys]: grad_out (M, c) (or (..., c) with keys.size leading rows) -> (n_rows, c)."""
    keys = np.asarray(keys).reshape(-1)
    go = np.asarray(grad_out, np.float32)
    go = go.reshape(keys.shape[0], go.shape[-1])
    f64, mag, d = _scatter64(keys, go.astype(np.float64), n_rows)
    return Scatter(f64, mag, d, index_put_f32(go, keys, n_rows, order))


def weighted_backward(grad_out, idx, w, n_rows: int, mode: str = "loop", order: str = "cuda") -> Scatter:
    """grad wrt feat of out[n] = sum_i feat[idx[n, i]] * w[n, i]; grad_out (n, c), idx / w (n, k).
    mode "loop": pointops.interpolation's k index_put results G_i, summed by autograd as ((G_(k-1) + G_(k-2)) + ...) + G_0;
    mode "sum": one index_put over all (n, i) in ascending n*k + i (torch.sum(index_points(p2, idx) * w, 2)).
    ``f32`` holds that float32 result; the float64 sum does not depend on the mode."""
    go = np.asarray(grad_out, np.float32)
    idx = np.asarray(idx).astype(np.int64)
    w = np.asarray(w, np.float32)
    n, k = idx.shape
    t64 = go.astype(np.float64)[:, None, :] * w.astype(np.float64)[:, :, None]            # (n, k, c)
    f64, mag, d = _scatter64(idx.reshape(-1), t64.reshape(n * k, -1), n_rows)
    t32 = go[:, None, :] * w[:, :, None]                                                   # float32 products, as torch rounds them
    if mode == "sum":
        f32 = index_put_f32(t32.reshape(n * k, -1), idx.reshape(-1), n_rows, order)
    else:
        f32 = None
        for i in range(k - 1, -1, -1):
            g = index_put_f32(t32[:, i], idx[:, i], n_rows, order)
            f32 = g if f32 is None else f32 + g
    return Scatter(f64, mag, d, f32)


def subtraction_backward(idx, grad_out, n2: int):
    """out[n, s] = in1[n] - in2[idx[n, s]]: (grad_in1, grad_in2) as Scatter; grad_out (n, ns, c)."""
    idx = np.asarray(idx).astype(np.int64)
    go = np.asarray(grad_out, np.float32).astype(np.float64)
    n, ns, c = go.shape
    g1 = Scatter(go.sum(1), np.abs(go).sum(1), np.full((n, c), ns))
    return g1, Scatter(*_scatter64(idx.reshape(-1), -go.reshape(n * ns, c), n2))


def aggregation_backward(inp, pos, w, idx, grad_out):
    """out[n, ch] = sum_s (inp[idx[n, s], ch] + pos[n, s, ch]) * w[n, s, ch % w_c]:
    (grad_input Scatter, grad_position float32 (exact: one product), grad_weight Scatter)."""
    inp = np.asarray(inp, np.float32)
    pos = np.asarray(pos, np.float32)
    w = np.asarray(w, np.float32)
    idx = np.asarray(idx).astype(np.int64)
    go = np.asarray(grad_out, np.float32)
    n, ns, c = pos.shape
    w_c = w.shape[-1]
    ch_w = np.arange(c) % w_c
    wf = w[:, :, ch_w]                                                                    # (n, ns, c)
    gp = go[:, None, :] * wf                                                              # float32 product
    gi = Scatter(*_scatter64(idx.reshape(-1), (go.astype(np.float64)[:, None, :] * wf.astype(np.float64)).reshape(n * ns, c),
                             inp.shape[0]))
    v = inp.astype(np.float64)[idx] + pos.astype(np.float64)                              # (n, ns, c)
    t = go.astype(np.float64)[:, None, :] * v
    f64 = np.zeros((n, ns, w_c))
    mag = np.zeros((n, ns, w_c))
    for j in range(w_c):
        f64[:, :, j] = t[:, :, j::w_c].sum(-1)
        mag[:, :, j] = np.abs(t[:, :, j::w_c]).sum(-1)
    d = np.broadcast_to(np.bincount(ch_w, minlength=w_c), (n, ns, w_c))
    return gi, gp, Scatter(f64, mag, d)


# -------------------------------------------------------------------------------------------------------------- forwards
def weighted_forward(inp, idx, w):
    """out[n] = sum_i inp[idx[n, i]] * w[n, i] in float64 -> (f64, mag, d)."""
    inp64 = np.asarray(inp, np.float32).astype(np.float64)
    idx = np.asarray(idx).astype(np.int64)
    t = inp64[idx] * np.asarray(w, np.float32).astype(np.float64)[:, :, None]
    return t.sum(1), np.abs(t).sum(1), np.full(t.shape[::2], idx.shape[1])


def aggregation_forward(inp, pos, w, idx):
    """out[n, ch] = sum_s (inp[idx[n, s], ch] + pos[n, s, ch]) * w[n, s, ch % w_c] in float64 -> (f64, mag, d = nsample).
    A float32 evaluation that rounds each inner sum and each product-add once errs by at most u * mag for the inner sums
    plus nsample * u * mag for the chain: (d + 1) * u * mag, the usual bound."""
    pos64 = np.asarray(pos, np.float32).astype(np.float64)
    n, ns, c = pos64.shape
    w64 = np.asarray(w, np.float32).astype(np.float64)
    v = np.asarray(inp, np.float32).astype(np.float64)[np.asarray(idx).astype(np.int64)] + pos64
    t = v * w64[:, :, np.arange(c) % w64.shape[-1]]
    return t.sum(1), np.abs(t).sum(1), np.full((n, c), ns)
