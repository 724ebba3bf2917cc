"""Float64 reference of one train step with a first-order error magnitude for every output element.

`rel_err` (largest absolute error over largest reference element) is blind to most of the target-table gradient: in
dY = P^T v the B target rows carry about |v| / B each and the other Y - B rows about |v| / Y, so a wrong softmax
normaliser or a zeroed non-target slab stays far below any usable tolerance.  This module computes each output in
float64 from the float32 parameters together with a magnitude M of the same shape, obtained by evaluating the same
formulas again on absolute values (x^ the value, M(.) its magnitude):

  * products and sums: M(A.B) = |A|.|B| for exact inputs (the float32 parameters and indices), otherwise
    M(A.B) = M(A).|B| + |A|.M(B) + |A.B| (the last term is the rounding of the result); subtractions add magnitudes;
  * tanh: M(h) = |h| + (1 - h^2) M(pre);
  * softmax / exp: the output carries a relative error equal to the magnitude of its argument, so
    M(alpha) = alpha (1 + M(z) + max_c M(z)), M(p) = p (1 + M(s) + max_y M(s)), M(dl) = (M(p) + |p - onehot|) / B;
  * the embedding scatters add M(dx) rows with np.add.at, so every gradient row is bounded at its own scale.

An implementation whose arithmetic has unit roundoff u then satisfies |got - ref| <= tau M element by element with tau
a small multiple of u.  The check adds 1e-30, so an element with M = 0 (a row only masked contexts reference, a masked
attention weight) must come out exactly 0.  In tf32 an element-wise bound loose enough for operand rounding no longer
sees a small systematic error, so tf32 is also held to normwise relative errors over named slices (`slice_errors`).

The head is evaluated in blocks of target rows so that no [B, Y] float64 array exists whole, and the context part in
blocks of examples; a train step at B = 1024, C = 200, Y = 261,246 needs about 3 GB.  Test infrastructure only.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict

import numpy as np

TAU_FP32 = 2e-6          # fp32 FFMA and 3xTF32: ~17 u32; the float32 numpy oracle stays below 1e-7
TAU_TF32 = 4e-3          # tf32: operands rounded to 10 mantissa bits, u = 2^-11 = 4.9e-4 per operand
SLICE_TOL_TF32 = 1e-2    # tf32 normwise relative error per slice
# fp32 FFMA and 3xTF32 normwise relative error per slice.  The float32 numpy oracle stays below 4e-6, and so does the
# engine everywhere except 3xTF32 at the production shape (B = 1024, C = 200, Y = 261,246), where tok, path, W and a
# reach 6.4e-5 on an H100 (fp32 FFMA: 5.2e-6; 3xTF32 at B = 1000, C = 50, Y = 5003: 3.1e-6).  1e-4 still catches a 0.1 %
# systematic error 10x over, where the element-wise bound lets about 0.2 % through on the non-target dY rows.
SLICE_TOL_FP32 = 1e-4
SLICE_TOL = {0: SLICE_TOL_FP32, 1: SLICE_TOL_TF32, 2: SLICE_TOL_FP32}     # by engine math mode


@dataclass
class Ref64:
    """Values (float64) and magnitudes of one step.  vals / mags hold v, alpha, dv and the five gradients; extra holds
    the per-example log-sum-exp "lse" and, for the full softmax, the smallest probability "pmin", the loss magnitude
    "loss_mag" and each row's largest log U = max_y s - s_true with its column ("log_umax", "umax_col")."""
    loss: float
    vals: Dict[str, np.ndarray]
    mags: Dict[str, np.ndarray]
    targets: np.ndarray                     # the target rows of the batch (dY target slice)
    extra: Dict[str, object] = field(default_factory=dict)


def _f64(params):
    return {k: np.asarray(v, dtype=np.float64) for k, v in params.items()}


def _keep_scale(keep, dropout_mask, rows):
    if dropout_mask is None or keep >= 1.0:
        return None
    # the engine and the float32 oracle both multiply by the float32 value of 1 / keep
    return dropout_mask[rows].astype(np.float64) * float(np.float32(1.0 / keep))


def _context_forward(P, src, pth, tgt, mask, ks):
    """Forward of a block of examples: x, h, alpha, v and their magnitudes."""
    E, C = src.shape
    tok, path, W, a = P["tok"], P["path"], P["W"], P["a"]
    x = np.concatenate([tok[src], path[pth], tok[tgt]], axis=-1).reshape(E * C, -1)
    Mx = np.zeros_like(x)
    if ks is not None:
        x = x * ks
        Mx = np.abs(x)                                  # the fp32 product x * (1 / keep) is rounded
    pre = x @ W
    Mpre = (Mx + np.abs(x)) @ np.abs(W) if ks is None else Mx @ np.abs(W) + np.abs(pre)
    h = np.tanh(pre)
    Mh = np.abs(h) + (1.0 - h * h) * Mpre
    z = (h @ a).reshape(E, C)
    Mz = (Mh @ np.abs(a)).reshape(E, C) + np.abs(z)
    valid = mask > 0
    with np.errstate(invalid="ignore"):
        zz = np.where(valid, z, -np.inf)
        e = np.exp(zz - zz.max(axis=1, keepdims=True))
        alpha = e / e.sum(axis=1, keepdims=True)
    Mzmax = np.where(valid, Mz, 0.0).max(axis=1, keepdims=True)
    Malpha = np.where(valid, alpha * (1.0 + Mz + Mzmax), 0.0)
    H, MH = h.reshape(E, C, -1), Mh.reshape(E, C, -1)
    v = np.einsum("bc,bcd->bd", alpha, H)
    Mv = np.einsum("bc,bcd->bd", Malpha, np.abs(H)) + np.einsum("bc,bcd->bd", alpha, MH) + np.abs(v)
    return dict(x=x, Mx=Mx, H=H, MH=MH, alpha=alpha, Malpha=Malpha, v=v, Mv=Mv)


def _context_backward(P, f, dv, Mdv, ks):
    """Backward of a block of examples from dv: (g_W, g_a, dx) and their magnitudes (oracle.backward line by line)."""
    W, a = P["W"], P["a"]
    aW, aa = np.abs(W), np.abs(a)
    H, MH, al, Mal = f["H"], f["MH"], f["alpha"], f["Malpha"]
    aH, adv = np.abs(H), np.abs(dv)
    E, C, D = H.shape
    dal = np.einsum("bcd,bd->bc", H, dv)
    Mdal = np.einsum("bcd,bd->bc", MH, adv) + np.einsum("bcd,bd->bc", aH, Mdv) + np.abs(dal)
    t = (al * dal).sum(axis=1, keepdims=True)
    Mt = (Mal * np.abs(dal) + al * Mdal).sum(axis=1, keepdims=True) + np.abs(t)
    r = dal - t
    Mr = Mdal + Mt + np.abs(r)
    dz = al * r
    Mdz = Mal * np.abs(r) + al * Mr + np.abs(dz)
    dh = al[:, :, None] * dv[:, None, :] + dz[:, :, None] * a
    Mdh = (Mal[:, :, None] * adv[:, None, :] + al[:, :, None] * Mdv[:, None, :] + Mdz[:, :, None] * aa
           + np.abs(dh))
    g = 1.0 - H * H
    du = (dh * g).reshape(E * C, D)
    Mdu = (Mdh * g + np.abs(dh) * 2.0 * aH * MH).reshape(E * C, D) + np.abs(du)
    g_a = np.einsum("bc,bcd->d", dz, H)
    Mg_a = np.einsum("bc,bcd->d", Mdz, aH) + np.einsum("bc,bcd->d", np.abs(dz), MH)     # |g_a| added by the caller
    x, Mx = f["x"], f["Mx"]
    g_W = x.T @ du
    Mg_W = Mx.T @ np.abs(du) + np.abs(x).T @ Mdu                                     # |g_W| added by the caller
    dx = du @ W.T
    Mdx = Mdu @ aW.T + np.abs(dx)
    if ks is not None:
        dx = dx * ks
        Mdx = Mdx * ks + np.abs(dx)
    return g_W, Mg_W, g_a, Mg_a, dx, Mdx


def _scatter(out, Mout, d, src, pth, tgt, dx, Mdx, which):
    """The three np.add.at scatters of oracle.backward (token table: which = "tok", path table: "path")."""
    if which == "tok":
        np.add.at(out, src.ravel(), dx[:, 0:d]); np.add.at(Mout, src.ravel(), Mdx[:, 0:d])
        np.add.at(out, tgt.ravel(), dx[:, 2 * d:]); np.add.at(Mout, tgt.ravel(), Mdx[:, 2 * d:])
    else:
        np.add.at(out, pth.ravel(), dx[:, d:2 * d]); np.add.at(Mout, pth.ravel(), Mdx[:, d:2 * d])


def forward64(params, src, pth, tgt, mask, ex_block=128):
    """Evaluation forward (no dropout): (v, Mv, alpha, Malpha)."""
    P = _f64(params)
    B = src.shape[0]
    out = {k: [] for k in ("v", "Mv", "alpha", "Malpha")}
    for b0 in range(0, B, ex_block):
        sl = slice(b0, min(B, b0 + ex_block))
        f = _context_forward(P, src[sl], pth[sl], tgt[sl], mask[sl], None)
        for k in out:
            out[k].append(f[k])
    return tuple(np.concatenate(out[k]) for k in ("v", "Mv", "alpha", "Malpha"))


def _lse_pass(Yt, v, Mv, y_block):
    """First pass over the target rows: log-sum-exp, max M(s), and each row's largest logit with its column."""
    B, Y = v.shape[0], Yt.shape[0]
    m = np.full(B, -np.inf)
    col = np.zeros(B, dtype=np.int64)
    ssum = np.zeros(B)
    Msmax = np.zeros(B)
    for y0 in range(0, Y, y_block):
        Yb = Yt[y0:y0 + y_block]
        s = v @ Yb.T
        Ms = Mv @ np.abs(Yb).T + np.abs(s)
        Msmax = np.maximum(Msmax, Ms.max(axis=1))
        bm, bi = s.max(axis=1), s.argmax(axis=1)
        col = np.where(bm > m, y0 + bi, col)
        mn = np.maximum(m, bm)
        ssum = ssum * np.exp(m - mn) + np.exp(s - mn[:, None]).sum(axis=1)
        m = mn
    return m + np.log(ssum), Msmax, m, col


def _loss_extra(lse, Mlse, s_true, Ms_true, smax, col):
    """extra entries of the loss: "lse"; "loss_mag", the mean over b of M(lse_b) + M(s_true,b), so that a loss whose
    logits are in the hundreds can be held to tau M rather than to a flat tolerance below its fp32 rounding; and per row
    "log_umax" = max_y s - s_true (the log of the exp_slab schedule's largest U = exp(s - s_true)) and "umax_col", its
    column."""
    return dict(lse=lse, loss_mag=float(np.mean(Mlse + Ms_true)), log_umax=smax - s_true, umax_col=col)


def head_loss64(params, v, target, Mv=None, y_block=16384):
    """Loss of the full softmax from given code vectors [B, D] (exact float32 values unless Mv is given): (loss, extra)
    with extra as _full_head's ("lse", "loss_mag", "log_umax", "umax_col")."""
    Yt = np.asarray(params["tgt"], dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    Mv = np.abs(v) if Mv is None else Mv
    lse, _, smax, col = _lse_pass(Yt, v, Mv, y_block)
    Mlse = np.abs(lse)
    for y0 in range(0, Yt.shape[0], y_block):
        Yb = Yt[y0:y0 + y_block]
        s = v @ Yb.T
        Mlse += (np.exp(s - lse[:, None]) * (Mv @ np.abs(Yb).T + np.abs(s))).sum(axis=1)
    s_true = np.einsum("bd,bd->b", v, Yt[target])
    Ms_true = np.einsum("bd,bd->b", Mv, np.abs(Yt[target])) + np.abs(s_true)
    return float(np.mean(lse - s_true)), _loss_extra(lse, Mlse, s_true, Ms_true, smax, col)


def _full_head(P, v, Mv, target, y_block, soft_factor=1.0):
    """Full softmax over Y in row blocks: loss, dv, dY and magnitudes.  Two passes (log-sum-exp and max M(s) first)."""
    Yt = P["tgt"]
    B, Y = v.shape[0], Yt.shape[0]
    av = np.abs(v)
    s_true = np.einsum("bd,bd->b", v, Yt[target])
    Ms_true = np.einsum("bd,bd->b", Mv, np.abs(Yt[target])) + np.abs(s_true)
    lse, Msmax, smax, col = _lse_pass(Yt, v, Mv, y_block)
    Mlse = np.abs(lse)
    loss = float(np.mean(lse - s_true))
    dv = np.zeros_like(v)
    Mdv = np.zeros_like(v)
    gY = np.empty_like(Yt)
    MgY = np.empty_like(Yt)
    pmin = np.inf
    rows = np.arange(B)
    for y0 in range(0, Y, y_block):
        Yb = Yt[y0:y0 + y_block]
        aYb = np.abs(Yb)
        s = v @ Yb.T
        Ms = Mv @ aYb.T + np.abs(s)
        p = np.exp(s - lse[:, None])
        pmin = min(pmin, float(p.min()))
        Mlse += (p * Ms).sum(axis=1)
        Mp = p * (1.0 + Ms + Msmax[:, None])
        q = p * soft_factor
        hit = (target >= y0) & (target < y0 + Yb.shape[0])
        q[rows[hit], target[hit] - y0] -= 1.0
        dl = q / B
        adl = np.abs(dl)
        Mdl = (Mp + np.abs(q)) / B
        gYb = dl.T @ v
        gY[y0:y0 + Yb.shape[0]] = gYb
        MgY[y0:y0 + Yb.shape[0]] = Mdl.T @ av + adl.T @ Mv + np.abs(gYb)
        dv += dl @ Yb
        Mdv += Mdl @ aYb
    Mdv += np.abs(dv)
    return loss, dv, Mdv, gY, MgY, dict(pmin=pmin, **_loss_extra(lse, Mlse, s_true, Ms_true, smax, col))


def _sampled_head(P, v, Mv, target, sampled, logq_true, logq_sampled):
    """oracle.sampled_softmax_loss_and_grads with magnitudes."""
    Yt = P["tgt"]
    B = v.shape[0]
    av = np.abs(v)
    tr, sr = Yt[target], Yt[sampled]
    lq_t, lq_s = logq_true.astype(np.float64), logq_sampled.astype(np.float64)
    l_true = np.einsum("bd,bd->b", v, tr) - lq_t
    Ml_true = np.einsum("bd,bd->b", Mv, np.abs(tr)) + np.abs(l_true)
    l_samp = v @ sr.T - lq_s[None, :]
    Ml_samp = Mv @ np.abs(sr).T + np.abs(l_samp)
    hit = sampled[None, :] == target[:, None]
    l_samp = np.where(hit, -1e9, l_samp)
    Ml_samp = np.where(hit, 0.0, Ml_samp)
    logits = np.concatenate([l_true[:, None], l_samp], axis=1)
    Ml = np.concatenate([Ml_true[:, None], Ml_samp], axis=1)
    mx = logits.max(axis=1, keepdims=True)
    lse = mx[:, 0] + np.log(np.exp(logits - mx).sum(axis=1))
    loss = float(np.mean(lse - logits[:, 0]))
    p = np.exp(logits - lse[:, None])
    Mp = p * (1.0 + Ml + Ml.max(axis=1, keepdims=True))
    q = p.copy()
    q[:, 0] -= 1.0
    dl = q / B
    Mdl = (Mp + np.abs(q)) / B
    dl_s = np.where(hit, 0.0, dl[:, 1:])
    Mdl_s = np.where(hit, 0.0, Mdl[:, 1:])
    adl0, Mdl0, adl_s = np.abs(dl[:, :1]), Mdl[:, :1], np.abs(dl_s)
    dv = dl[:, :1] * tr + dl_s @ sr
    Mdv = Mdl0 * np.abs(tr) + Mdl_s @ np.abs(sr) + np.abs(dv)
    gY = np.zeros_like(Yt)
    MgY = np.zeros_like(Yt)
    np.add.at(gY, target, dl[:, :1] * v)
    np.add.at(MgY, target, Mdl0 * av + adl0 * Mv + np.abs(dl[:, :1] * v))
    gs = dl_s.T @ v
    np.add.at(gY, sampled, gs)
    np.add.at(MgY, sampled, Mdl_s.T @ av + adl_s.T @ Mv + np.abs(gs))
    return loss, dv, Mdv, gY, MgY, dict(lse=lse)


def train_step64(params, src, pth, tgt, mask, target, *, keep=1.0, dropout_mask=None, sampled=None, logq_true=None,
                 logq_sampled=None, y_block=16384, ex_block=64, soft_factor=1.0) -> Ref64:
    """One train step (full softmax, or the sampled softmax when `sampled` is given) in float64 with magnitudes.
    dropout_mask: [B * C, 3 d] 0/1 (oracle.dropout_keep_mask) applied with `keep` as the engine and oracle do.
    soft_factor scales the softmax part of dL/dlogits (the one-hot part intact): 1 except in the tests of this check."""
    P = _f64(params)
    B, C = src.shape
    d = P["tok"].shape[1]
    vs, Mvs, als, Mals = [], [], [], []
    for b0 in range(0, B, ex_block):
        sl = slice(b0, min(B, b0 + ex_block))
        rows = np.arange(sl.start * C, sl.stop * C)
        f = _context_forward(P, src[sl], pth[sl], tgt[sl], mask[sl], _keep_scale(keep, dropout_mask, rows))
        vs.append(f["v"]); Mvs.append(f["Mv"]); als.append(f["alpha"]); Mals.append(f["Malpha"])
    v, Mv = np.concatenate(vs), np.concatenate(Mvs)
    if sampled is None:
        loss, dv, Mdv, gY, MgY, extra = _full_head(P, v, Mv, target, y_block, soft_factor)
    else:
        loss, dv, Mdv, gY, MgY, extra = _sampled_head(P, v, Mv, target, sampled, logq_true, logq_sampled)
    g = {k: np.zeros_like(P[k]) for k in ("tok", "path", "W", "a")}
    Mg = {k: np.zeros_like(P[k]) for k in ("tok", "path", "W", "a")}
    for b0 in range(0, B, ex_block):
        sl = slice(b0, min(B, b0 + ex_block))
        rows = np.arange(sl.start * C, sl.stop * C)
        ks = _keep_scale(keep, dropout_mask, rows)
        f = _context_forward(P, src[sl], pth[sl], tgt[sl], mask[sl], ks)
        gW, MgW, ga, Mga, dx, Mdx = _context_backward(P, f, dv[sl], Mdv[sl], ks)
        g["W"] += gW; Mg["W"] += MgW
        g["a"] += ga; Mg["a"] += Mga
        _scatter(g["tok"], Mg["tok"], d, src[sl], pth[sl], tgt[sl], dx, Mdx, "tok")
        _scatter(g["path"], Mg["path"], d, src[sl], pth[sl], tgt[sl], dx, Mdx, "path")
    Mg["W"] += np.abs(g["W"])
    Mg["a"] += np.abs(g["a"])
    vals = dict(v=v, alpha=np.concatenate(als), dv=dv, tgt=gY, **g)
    mags = dict(v=Mv, alpha=np.concatenate(Mals), dv=Mdv, tgt=MgY, **Mg)
    return Ref64(loss, vals, mags, np.unique(target), extra)


def example_dx64(params, src, pth, tgt, mask, dv, b, *, keep=1.0, dropout_mask=None):
    """dX [C, 3 d] of example b given the step's dv [B, D]: what each of its contexts scatters into the tables."""
    P = _f64(params)
    C = src.shape[1]
    sl = slice(b, b + 1)
    ks = _keep_scale(keep, dropout_mask, np.arange(b * C, (b + 1) * C))
    f = _context_forward(P, src[sl], pth[sl], tgt[sl], mask[sl], ks)
    return _context_backward(P, f, dv[sl], np.zeros_like(dv[sl]), ks)[4]


def topk64(params, v, Mv, k, y_block=16384):
    """Float64 evaluation scores s = v . Y^T (oracle.evaluate_topk) from a code-vector reference (v, Mv), in blocks of
    target rows: the top min(k + 1, Y) scores per row, sorted descending, with their row indices and magnitudes
    M(s) = M(v).|Y|^T + |s|, and the probabilities softmax(s) of those rows with M(p) = p (1 + M(s) + max_y M(s))
    (normalize = 2).  Returns dict(idx, s, Ms, p, Mp), each [B, min(k + 1, Y)]."""
    Yt = np.asarray(params["tgt"], dtype=np.float64)
    B, Y = v.shape[0], Yt.shape[0]
    kk = min(k + 1, Y)
    best_s = np.empty((B, 0))
    best_i = np.empty((B, 0), dtype=np.int64)
    m = np.full(B, -np.inf)
    ssum = np.zeros(B)
    Msmax = np.zeros(B)
    for y0 in range(0, Y, y_block):
        Yb = Yt[y0:y0 + y_block]
        s = v @ Yb.T
        Msmax = np.maximum(Msmax, (Mv @ np.abs(Yb).T + np.abs(s)).max(axis=1))
        mn = np.maximum(m, s.max(axis=1))
        ssum = ssum * np.exp(m - mn) + np.exp(s - mn[:, None]).sum(axis=1)
        m = mn
        cs = np.concatenate([best_s, s], axis=1)
        ci = np.concatenate([best_i, np.broadcast_to(np.arange(y0, y0 + Yb.shape[0]), s.shape)], axis=1)
        part = np.argpartition(-cs, kk - 1, axis=1)[:, :kk]
        best_s, best_i = np.take_along_axis(cs, part, axis=1), np.take_along_axis(ci, part, axis=1)
    order = np.lexsort((best_i, -best_s), axis=1)                # descending, ties to the lower index
    s, idx = np.take_along_axis(best_s, order, axis=1), np.take_along_axis(best_i, order, axis=1)
    Ms = np.einsum("bd,bkd->bk", Mv, np.abs(Yt[idx])) + np.abs(s)
    lse = m + np.log(ssum)
    p = np.exp(s - lse[:, None])
    Mp = p * (1.0 + Ms + Msmax[:, None])
    return dict(idx=idx, s=s, Ms=Ms, p=p, Mp=Mp)


LOG_U_EDGE = float(np.log(5e29))     # just inside the exp_slab window's largest U, 1e30


def _row_logits_max(Yt, v, exclude, y_block=16384):
    """max_y v_b . Y_y over y != exclude[b], per row of v."""
    out = np.full(v.shape[0], -np.inf)
    rows = np.arange(v.shape[0])
    for y0 in range(0, Yt.shape[0], y_block):
        s = v @ Yt[y0:y0 + y_block].T
        hit = (exclude >= y0) & (exclude < y0 + s.shape[1])
        s[rows[hit], exclude[hit] - y0] = -np.inf
        out = np.maximum(out, s.max(axis=1))
    return out


def _column_direction(v, b):
    """u with v_b . u = 1 and the other code vectors as orthogonal to it as they can be (ridge least squares)."""
    others = np.delete(v, b, axis=0)
    G = others.T @ others
    u = np.linalg.solve(G + 1e-3 * np.trace(G) / G.shape[0] * np.eye(G.shape[0]), v[b])
    return u / (v[b] @ u)


def quiet_row(v, candidates=64):
    """The example among the first `candidates` whose raise_column direction the other code vectors overlap least."""
    v = np.asarray(v, dtype=np.float64)
    leak = [np.abs(np.delete(v, b, axis=0) @ _column_direction(v, b)).max() for b in range(min(candidates, len(v)))]
    return int(np.argmin(leak))


def raise_column(params, v, target, b, col, log_u):
    """Copy of params in which example b's logit in column `col` exceeds its true-class logit by log_u, and the other
    examples' logits there move as little as possible: target row `col` moves along u, the least-squares solution of
    v_b . u = 1 with the other code vectors as orthogonal to u as they can be.  v: the step's code vectors [B, D] (after
    dropout).  No example may have `col` as its class."""
    assert not np.any(target == col), col
    v = np.asarray(v, dtype=np.float64)
    u = _column_direction(v, b)
    Yt = np.asarray(params["tgt"], dtype=np.float64)
    lam = log_u + v[b] @ Yt[target[b]] - v[b] @ Yt[col]
    out = dict(params)
    out["tgt"] = params["tgt"].copy()
    out["tgt"][col] = (Yt[col] + lam * u).astype(np.float32)
    return out


def rows_to_lower(v, target, n, candidates=256):
    """`n` examples for lower_true_rows: among the first `candidates` whose class no other example has, those whose
    raise_column direction the other code vectors overlap least."""
    v = np.asarray(v, dtype=np.float64)
    own = np.flatnonzero(np.bincount(target)[target] == 1)[:candidates]
    leak = [np.abs(np.delete(v, b, axis=0) @ _column_direction(v, b)).max() for b in own]
    return np.sort(own[np.argsort(leak, kind="stable")[:n]])


def lower_true_rows(params, v, target, rows, log_u, iters=4, y_block=16384):
    """Copy of params in which each example b of `rows` has its largest exp(s - s_true) at exp(log_u): its true-class row
    moves by -lambda_b u_b (u_b as in raise_column: v_b . u_b = 1, the other code vectors nearly orthogonal), which lowers
    s_true,b by lambda_b and the other examples' logits in that column by little.  The classes of `rows` must be
    distinct and no other example's, so no other true-class logit moves.  lambda is refined `iters` times, because
    lowering one row's class can raise another chosen row's largest logit a little."""
    rows = np.asarray(rows)
    t = target[rows]
    assert len(np.unique(t)) == len(rows) and not np.isin(np.delete(target, rows), t).any()
    v = np.asarray(v, dtype=np.float64)
    U = np.stack([_column_direction(v, b) for b in rows])
    vr = v[rows]
    Yt = np.asarray(params["tgt"], dtype=np.float64).copy()
    for _ in range(iters):
        gap = _row_logits_max(Yt, vr, t, y_block) - np.einsum("bd,bd->b", vr, Yt[t])
        Yt[t] -= (log_u - gap)[:, None] * U
    out = dict(params)
    out["tgt"] = params["tgt"].copy()
    out["tgt"][t] = Yt[t].astype(np.float32)
    return out


def tf32_truncate(a):
    """The tf32 operand the tensor cores read from an fp32 value: the low 13 mantissa bits dropped (truncation)."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def tf32_model_loss(params, src, pth, tgt, mask, target, *, keep=1.0, dropout_mask=None, y_block=16384,
                    true_logit="fp32"):
    """Loss of a train step whose two loss-bearing GEMMs read tf32-truncated operands, everything else exact: the
    context projection X.W and the logits v.Y^T.  true_logit: "fp32" keeps the true-class logit exact, as the exp_slab
    and recompute_logits schedules compute it (a separate fp32 dot product); "tf32" takes it from the truncated logits,
    as the two-pass and loader schedules do (they read it from the tensor-core slab).  Truncation biases every product
    toward zero, and a bias does not average out over the batch, so this is what tf32 converges to where the logits are
    large or have few terms; the float64 loss is what fp32 converges to."""
    assert true_logit in ("fp32", "tf32"), true_logit
    P = _f64(params)
    B, C = src.shape
    x = np.concatenate([P["tok"][src], P["path"][pth], P["tok"][tgt]], axis=-1).reshape(B * C, -1)
    ks = _keep_scale(keep, dropout_mask, np.arange(B * C))
    if ks is not None:
        x = (x.astype(np.float32) * np.float32(1.0 / keep)) * dropout_mask.astype(np.float32)
    h = np.tanh(tf32_truncate(x) @ tf32_truncate(P["W"]))
    z = np.where(mask > 0, (h @ P["a"]).reshape(B, C), -np.inf)
    with np.errstate(invalid="ignore"):
        al = np.exp(z - z.max(axis=1, keepdims=True))
        al /= al.sum(axis=1, keepdims=True)
    v = np.einsum("bc,bcd->bd", al, h.reshape(B, C, -1))
    vt = tf32_truncate(v)
    m = np.full(B, -np.inf)
    ssum = np.zeros(B)
    for y0 in range(0, P["tgt"].shape[0], y_block):
        s = vt @ tf32_truncate(P["tgt"][y0:y0 + y_block]).T
        mn = np.maximum(m, s.max(axis=1))
        ssum = ssum * np.exp(m - mn) + np.exp(s - mn[:, None]).sum(axis=1)
        m = mn
    if true_logit == "tf32":
        s_true = np.einsum("bd,bd->b", vt, tf32_truncate(P["tgt"][target]))
    else:
        s_true = np.einsum("bd,bd->b", v, P["tgt"][target])
    return float(np.mean(m + np.log(ssum) - s_true))


# ---- checks -----------------------------------------------------------------------------------------------------------

def err_ratio(got, ref, M):
    """(max err / M, flat index of the worst element); +inf marks an element with M = 0 and err > 0."""
    err = np.abs(np.asarray(got, dtype=np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0.0, 0.0, err / M)
    r = np.where(np.isnan(r), np.inf, r)
    i = int(np.argmax(r))
    return float(r.flat[i]), i


def check_elementwise(name, got, ref, M, tau):
    """|got - ref| <= tau M + 1e-30 for every element; returns max err / M for the test log."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = np.abs(got - ref)
    bad = ~(err <= tau * M + 1e-30)
    worst, i = err_ratio(got, ref, M)
    if bad.any():
        j = int(np.flatnonzero(bad)[np.argmax((err / np.maximum(M, 1e-300)).flat[np.flatnonzero(bad)])])
        idx = np.unravel_index(j, ref.shape)
        raise AssertionError("%s: %d of %d elements exceed tau = %.1e; worst at %s (row %d): got %.9g, ref %.9g, M %.3g; "
                             "max err/M %.3g" % (name, int(bad.sum()), bad.size, tau, tuple(int(x) for x in idx),
                                                 int(idx[0]), got.flat[j], ref.flat[j], M.flat[j], worst))
    return worst


def normwise(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    den = np.linalg.norm(ref)
    return float(np.linalg.norm(np.asarray(got, dtype=np.float64) - ref) / (den if den > 0 else 1.0))


def slice_errors(got: Dict[str, np.ndarray], ref: Ref64, names=("tok", "path", "W", "a", "v", "alpha", "dv")):
    """Normwise relative errors over the named slices present in `got`: dY target rows (tgt:target), dY non-target rows
    (tgt:other), and each whole tensor in `names`."""
    out = {}
    if "tgt" in got:
        Y = ref.vals["tgt"].shape[0]
        is_t = np.zeros(Y, bool)
        is_t[ref.targets] = True
        out["tgt:target"] = normwise(got["tgt"][is_t], ref.vals["tgt"][is_t])
        out["tgt:other"] = normwise(got["tgt"][~is_t], ref.vals["tgt"][~is_t])
    for k in names:
        if k in got:
            out[k] = normwise(got[k], ref.vals[k])
    return out


def check_slices(got, ref: Ref64, tol=SLICE_TOL_TF32, names=("tok", "path", "W", "a", "v", "alpha", "dv")):
    errs = slice_errors(got, ref, names)
    bad = {k: e for k, e in errs.items() if not e <= tol}
    assert not bad, "normwise slice errors over %.1e: %s (all: %s)" % (tol, bad, errs)
    return errs


def check_step(got: Dict[str, np.ndarray], ref: Ref64, tau, slice_tol=None, label=""):
    """Element-wise check of every tensor in `got` (names of Ref64.vals), plus the normwise slice checks at `slice_tol`
    when given.  Returns {name: max err / M} (and the slice errors under "slice:<name>")."""
    out = {}
    for k, a in got.items():
        out[k] = check_elementwise("%s%s" % (label, k), a, ref.vals[k], ref.mags[k], tau)
    if slice_tol is not None:
        for k, e in check_slices(got, ref, slice_tol).items():
            out["slice:" + k] = e
    return out
