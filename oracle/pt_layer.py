"""oracle/pt_layer.py -- float64 restatement of one ``tgn_pt_layer_forward`` launch (TEST INFRASTRUCTURE ONLY).

Keyword names are the descriptor's field names (include/tgn_b200.h, tgn_pt_layer_t); tensors are CPU tensors.  ``batch_sums``
is what passes 0-2 accumulate (the fp64 {sum, sumsq} over all n * K rows of t, w0 and w1), ``output`` what pass 3 writes,
``running_update`` the momentum update of the last launch.  A BatchNorm in mode 1 normalises with the ``stats_*`` it is given
(the kernel's own sums, so each pass is checked on its own) and, when that is None, with the sums this module computes.

The gathers and ``rel = p[nbr] - p[i]`` are float32, as in the kernel; the order of operations is the file header's
(csrc/pt_layer.cu), with channel ch reading share column ``ch % (c / 8)`` (blocks.py:43).  With ``dtype=torch.float64``
everything after the gathers is float64 and every value carries a first-order bound on the error of a float32 evaluation
of the same steps (u = 2^-24), propagated alongside it because batch-statistics scales can be far above 1:
* a product-and-sum of d terms (the bias one of them): (d + 1) u sum|terms|, plus the input's bound mapped through |W|;
* ``w0 = (xk - xq) + pr``: two roundings, u (|xk - xq| + |w0|);
* BatchNorm + ReLU as the kernel evaluates it, ``((x - mean_hi) - mean_lo) * scale + beta`` with a float32 scale:
  |scale| err(x) + u (5 |x - mean| |scale| + |beta|) (two subtractions, the scale, the product and the add; ReLU is
  1-Lipschitz);
* softmax over K with logit errors at most delta in its column: every weight a_j is off by a relative 2 delta, plus the
  rounding of l_j - max (u |l_j - max|), expf (2 ulp, 4u), the K-term sum and the division ((K + 4) u in all); with the
  rounding of v = xv + pr (u) and a K-term product-sum (K u), ``|d out| <= sum_j a_j err(pr_j) + sum_j a_j |v_j| (2 delta
  + (2K + 5) u + u |l_j - max|)``.  The CTA schedule's per-warp chains plus the sum of eight partials are at most K deep too;
* sums over the rows: ``|S_got - S| <= sum err(y)`` and ``|Q_got - Q| <= sum (2|y| + err(y)) err(y)``, each plus
  n K 2^-52 sum|.| for the fp64 accumulation (y * y of a float is exact in double).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import pw_chain

_F64 = torch.float64
U = 2.0 ** -24
_TAGS = ("p", "a", "b")
ROW_CHUNK = 1 << 21                     # query rows x K x c per chunk: ~16 MB per float64 tensor


def _affine(f: dict, i: int, stats) -> tuple:
    """(mean, scale, beta) of BatchNorm i (0 = p, 1 = a, 2 = b) in float64"""
    tag = _TAGS[i]
    cn = 3 if i == 0 else (f["c"] if i == 1 else f["c"] // 8)
    return pw_chain._bn_scale(int(f["bn_mode"][i]), cn, stats, float(f["n"]) * f["K"], f.get(tag + "_gamma"),
                              f.get(tag + "_beta"), f.get(tag + "_eps", 1e-5), f.get(tag + "_rmean"), f.get(tag + "_rvar"))


def _bn_relu(x, e, aff):
    mean, scale, beta = aff
    if x.dtype == torch.float32:                    # the kernel's split mean and float32 scale
        hi = mean.float()
        lo = (mean - hi.double()).float()
        y = ((x - hi) - lo) * scale.float() + beta.float()
    else:
        y = (x - mean) * scale + beta
    y = y.clamp(min=0.0)
    if e is None:
        return y, None
    sa = scale.abs()
    return y, sa * e + U * (5.0 * (x - mean).abs() * sa + beta.abs())


def _lin(x, e, w, b, bound: bool):
    w, b = w.to(x.dtype), b.to(x.dtype)
    y = x @ w.t() + b
    if not bound:
        return y, None
    wa = w.abs()
    eb = (w.shape[1] + 1) * U * (x.abs() @ wa.t() + b.abs())
    return y, eb if e is None else eb + e @ wa.t()


def _chain(f: dict, q: torch.Tensor, stage: int, affs, dt):
    """stage 0 -> (t, err); 1 -> (w0, err); 2 -> (w1, err); 3 -> (out, err) for the queries q"""
    bound = dt == _F64
    nbr = f["idx"][q].long()                                                   # (m, K)
    p = f["p"].float()
    rel = (p[nbr] - p[q].unsqueeze(1)).to(dt)                                  # float32 subtraction, as queryandgroup
    t, e = _lin(rel, None, f["p_w0"], f["p_b0"], bound)
    if stage == 0:
        return t, e
    tn, e = _bn_relu(t, e, affs[0])
    pr, epr = _lin(tn, e, f["p_w1"], f["p_b1"], bound)
    if stage == 3:
        xv = f["xv"].to(dt)[nbr]
    dk = f["xk"].to(dt)[nbr] - f["xq"].to(dt)[q].unsqueeze(1)
    w0 = dk + pr
    e = epr + U * (dk.abs() + w0.abs()) if bound else None
    if stage == 1:
        return w0, e
    ua, e = _bn_relu(w0, e, affs[1])
    w1, e = _lin(ua, e, f["a_w"], f["a_b"], bound)
    if stage == 2:
        return w1, e
    v1, e = _bn_relu(w1, e, affs[2])
    lg, el = _lin(v1, e, f["b_w"], f["b_b"], bound)                            # (m, K, c/8) logits
    mx = lg.amax(1, keepdim=True)
    ex = torch.exp(lg - mx)
    a = ex / ex.sum(1, keepdim=True)                                           # softmax over the K neighbours
    v = xv + pr
    share = f["c"] // (f["c"] // 8)                                            # channel ch reads column ch % (c/8)
    out = (v * a.repeat(1, 1, share)).sum(1)
    if not bound:
        return out, None
    K = f["K"]
    rho = 2.0 * el.amax(1, keepdim=True) + (2 * K + 5) * U + U * (lg - mx).abs()
    ar = a.repeat(1, 1, share)
    return out, (ar * epr).sum(1) + (ar * v.abs() * rho.repeat(1, 1, share)).sum(1)


def _chunks(f: dict, queries: torch.Tensor):
    step = max(1, ROW_CHUNK // (f["K"] * f["c"]))
    for s in range(0, queries.numel(), step):
        yield queries[s:s + step]


def batch_sums(*, passes: Optional[Sequence[int]] = None, dtype=_F64, **f) -> dict:
    """{Sigma, Sigma^2} over all n K rows of t (pass 0, BatchNorm_p), w0 (pass 1, _a) and w1 (pass 2, _b) -> {tag: (sums
    (2 cn,) float64, bound (2 cn,) float64 or None)} for ``passes`` (default: the BatchNorms in mode 1).  An earlier
    BatchNorm in mode 1 uses ``stats_<tag>`` when given, else the sums computed here."""
    if passes is None:
        passes = [i for i in range(3) if int(f["bn_mode"][i]) == 1]
    stats = [f.get("stats_" + t) for t in _TAGS]
    res = {}
    queries = torch.arange(f["n"])
    for k in range(max(passes, default=-1) + 1):
        if k not in passes and (stats[k] is not None or int(f["bn_mode"][k]) != 1):
            continue
        affs = [_affine(f, i, stats[i]) for i in range(k)]
        s1 = s2 = e1 = e2 = a1 = a2 = 0.0
        for q in _chunks(f, queries):
            y, e = _chain(f, q, k, affs, dtype)
            y = y.to(_F64)
            s1 = s1 + y.sum((0, 1))
            s2 = s2 + (y * y).sum((0, 1))
            if e is not None:
                e1 = e1 + e.sum((0, 1))
                e2 = e2 + ((2.0 * y.abs() + e) * e).sum((0, 1))
                a1 = a1 + y.abs().sum((0, 1))
                a2 = a2 + (y * y).sum((0, 1))
        sums = torch.cat([s1, s2])
        acc = float(f["n"]) * f["K"] * 2.0 ** -52
        bound = torch.cat([e1 + acc * a1, e2 + acc * a2]) if dtype == _F64 else None
        if stats[k] is None:
            stats[k] = sums
        if k in passes:
            res[_TAGS[k]] = (sums, bound)
    return res


def output(*, select=None, dtype=_F64, **f):
    """What pass 3 writes -> (out, bound), (n, c) or (len(select), c) for the queries ``select``, in that order; bound is
    None unless dtype is float64.  Every BatchNorm in mode 1 needs its stats_<tag> (missing ones are computed here)."""
    need = [i for i in range(3) if int(f["bn_mode"][i]) == 1 and f.get("stats_" + _TAGS[i]) is None]
    if need:
        f = dict(f)
        for tag, (s, _) in batch_sums(passes=need, **f).items():
            f["stats_" + tag] = s
    affs = [_affine(f, i, f.get("stats_" + _TAGS[i])) for i in range(3)]
    queries = torch.arange(f["n"]) if select is None else torch.as_tensor(select, dtype=torch.int64).reshape(-1)
    outs, bounds = [], []
    for q in _chunks(f, queries):
        o, e = _chain(f, q, 3, affs, dtype)
        outs.append(o)
        bounds.append(e)
    return torch.cat(outs), (torch.cat(bounds) if dtype == _F64 else None)


CASES = ("plain", "hard", "saturated", "uniform")


def make_case(c: int, K: int, p: torch.Tensor, idx: torch.Tensor, kind: str = "plain", seed: int = 0) -> dict:
    """Descriptor fields (CPU float32 tensors, bn_mode [1, 1, 1], update_running 1) of a layer over the cloud p (n, 3) with
    neighbourhoods idx (n, K).  kind:
    * plain: unit-scale features, BatchNorm weights in [0.5, 1.5);
    * hard: xk offset on every fourth channel (|mean| / std ~ 100 and ~ 1000 at BatchNorm_a, what a linear_k bias does),
      p_b0 and a_b offset (~ 10^3 at BatchNorm_p, ~ 300 std at BatchNorm_b), negative gamma on every third channel, one
      zero-variance channel per BatchNorm, eps = 1e-3 at BatchNorm_a, momentum 0.01 at _p and 1.0 at _b; running
      statistics near the batch ones so that mode 2 stays in range;
    * saturated: logits x 100 (near one-hot softmax);
    * uniform: b_w = 0 (exactly uniform softmax)."""
    assert kind in CASES
    n, cs = p.shape[0], c // 8
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)                                 # noqa: E731
    f = {"n": n, "c": c, "K": K, "p": p.float().contiguous(), "idx": idx.to(torch.int32).contiguous(),
         "xq": r(n, c), "xk": r(n, c), "xv": r(n, c),
         "p_w0": r(3, 3), "p_b0": r(3) * 0.01, "p_w1": r(c, 3) / 3 ** 0.5, "p_b1": r(c) * 0.1,
         "a_w": r(cs, c) / c ** 0.5, "a_b": r(cs) * 0.1, "b_w": r(cs, cs) / cs ** 0.5, "b_b": r(cs) * 0.1,
         "bn_mode": [1, 1, 1], "update_running": 1}
    for tag, cn in (("p", 3), ("a", c), ("b", cs)):
        f.update({tag + "_gamma": torch.rand(cn, generator=g) + 0.5, tag + "_beta": r(cn) * 0.1,
                  tag + "_rmean": r(cn) * 0.1, tag + "_rvar": torch.rand(cn, generator=g) + 0.5,
                  tag + "_eps": 1e-5, tag + "_momentum": 0.1})
    if kind == "hard":
        nbr = f["idx"].long()
        t = (f["p"][nbr] - f["p"].unsqueeze(1)).reshape(-1, 3).double() @ f["p_w0"].double().t()
        f["p_w0"][2] = 0.0                                                      # t[2] = p_b0[2] on every row
        f["p_b0"][0] += float(1e3 * t[:, 0].std()) if t.shape[0] > 1 else 1.0
        f["p_rmean"] = (t.mean(0) + f["p_b0"].double()).float()
        f["p_rvar"] = (t.var(0, unbiased=False) + 1e-4).float() if t.shape[0] > 1 else f["p_rvar"]
        f["xk"][:, 0::8] += 140.0
        f["xk"][:, 4::8] += 1400.0
        f["a_rmean"][0::8] += 140.0
        f["a_rmean"][4::8] += 1400.0
        f["xk"][:, 3] = f["xq"][:, 3] = 0.5                                     # w0[3] = p_b1[3] on every row
        f["p_w1"][3] = 0.0
        f["a_b"][0] += 300.0
        f["b_rmean"][0] += 300.0
        if cs > 1:
            f["a_w"][1] = 0.0                                                   # w1[1] = a_b[1] on every row
        for tag in ("p", "a", "b"):
            f[tag + "_gamma"][1::3] *= -1.0
        f.update(a_eps=1e-3, p_momentum=0.01, b_momentum=1.0)
    elif kind == "saturated":
        f["b_w"] *= 100.0
        f["b_b"] *= 100.0
    elif kind == "uniform":
        f["b_w"].zero_()
    return f


def running_update(**f) -> dict:
    """torch's momentum update of the launch -> {tag: (running_mean, running_var) float64} for every BatchNorm whose
    buffers it changes (mode 1, both running pointers set, update_running != 0), from stats_<tag>"""
    res = {}
    if not int(f.get("update_running", 0)):
        return res
    for i, tag in enumerate(_TAGS):
        rm, rv = f.get(tag + "_rmean"), f.get(tag + "_rvar")
        if int(f["bn_mode"][i]) != 1 or rm is None or rv is None:
            continue
        res[tag] = pw_chain.running_update(f["stats_" + tag], float(f["n"]) * f["K"], f.get(tag + "_momentum", 0.1), rm, rv)
    return res
