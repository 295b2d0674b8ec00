"""The LayerNorm-normalising GEMM epilogues (the ``LNF`` instantiations of vx_gemm.cu) against an fp64 reference, element
by element, under an error bound a correct kernel cannot exceed; then against the operation itself, LayerNorm -> Linear,
under the bound of the default path (LayerNorm kernel, then GEMM); then the UNet blocks under VX_LN_FOLD / VX_LN_FUSE.

    lnfold   ops.gemm_lnfold    out = s (r (A wf^T - mu colsum) + bf + b2[m // div]) + res, (mu, r) from ops.row_stats
    lnparts  ops.gemm_lnparts   the same epilogue, (mu, r) rebuilt in the kernel from ops.gemm_rowsums' partial slots
    gemm_ln  ops.gemm_ln        the same epilogue, (mu, r) from the row tile resident in shared memory (two passes)
    rowsums  ops.gemm_rowsums   the producer: ops.gemm's linear epilogue plus per-row partial (sum h, sum h^2) slots

wf = bf16(gamma w), colsum = sum_k wf (fp32, of the ROUNDED weights), bf = w beta + b (ops.fold_layernorm).  u = 2^-24 is the
fp32 unit roundoff.

1. Kernel against its own arithmetic (``lnfold_ref64``).  The reference takes exactly the bf16 / fp32 operands the kernel
read and a reference (mu, r) with absolute uncertainties (d_mu, d_r) of the statistics source.  Per output element, with
P = |A| |wf|^T and t = A wf^T - mu colsum:

    d_t = K 2^-22 P + 2^-22 (P + |mu colsum|) + |colsum| d_mu
    d_z = r d_t + d_r (|t| + d_t)                                  (z = r t;  |r' t' - r t| <= r |t' - t| + |r' - r| |t'|)
    |out - ref| <= 2^-8 |ref| + |s| d_z + 2^-20 ref_abs,   ref_abs = |s| (|z| + d_z + |bf| + |b2|) + |res|

* K 2^-22 P: the bf16 x bf16 products are exact in fp32; K of them summed in fp32 move the sum by at most K u P, x 2 for
  tensor-core adds that may truncate instead of round, x 2 for the order of the partial sums across k-steps and K blocks
  (the GEMM bound of tests/test_gemm_bounds_gpu.py).  P runs over the UNCENTRED row: this is where the fold pays for
  |mean| / sigma (below).
* 2^-22 (P + |mu colsum|): the product mu colsum and the subtraction from the accumulator (one fma, or two roundings),
  each u of a value no larger than P + |mu colsum|, x 2 for the two roundings, x 2 again for the fma's contraction order.
* |colsum| d_mu and d_r (|t| + d_t): the statistics the kernel used, against the reference's.
* 2^-20 ref_abs: r * t, + bf, + b2, * s, + res: a few fp32 roundings, each u of a value no larger than ref_abs.
* 2^-8 |ref|: the one rounding of the output to bf16 (unit roundoff 2^-8 at 8 significant bits).
GEGLU: V and G are two such columns (each with its own colsum: sv, sg), d_V = d_z_V + 2^-22 (|z_V| + |b_V|) (the r * t and
+ b roundings) and likewise d_G, propagated through V gelu(G) by tests/test_gemm_bounds_gpu.geglu_propagate.

The statistics sources:
* lnfold: the (mu, r) array the kernel read: d_mu = d_r = 0, the check is of the epilogue alone.
* lnparts: the reference rebuilds S1 = sum_j p_j.x, S2 = sum_j p_j.y in fp64 from the nparts slots the kernel read, in slot
  order, mu = S1 / K, v = max(S2 / K - mu^2, 0).  The kernel sums the slots in fp32 ((nparts - 1) adds: nparts u sum_j
  |p_j|) and multiplies by fp32(1 / K) (two more u), so
      d_mu = nparts u sum_j |p_j.x| / K + 2 u |mu|,   d_E2 = (nparts + 2) u S2 / K,
      d_v  = d_E2 + 2 |mu| d_mu + d_mu^2 + 2 u (S2 / K + mu^2) + u (v + eps)
  the third term is the s2 / K - mu^2 cancellation (one fma rounding, and the clamp at 0 can only move the value toward v),
  the last the rounding of v + eps.  With x = d_v / (v + eps) the relative rstd error is (1 - x)^-1/2 - 1 (~ x / 2 =
  d_v / (2 (v + eps)) when small) plus 2^-22 for rsqrtf (2 ulp); x >= 1 leaves rstd unbounded (the row's d_r is infinite:
  the bound makes no claim there, section 2 shows what such rows get).
* gemm_ln: the reference is the fp64 two-pass mean / rstd of the row, with twice the bound of
  tests/test_norm_bounds_gpu.row_stats_ref64 (2^-17 max|x| for the mean, 2^-18 r + 2^-17 max|x| r^2 for rstd).  That bound is
  derived for 64 sequential adds per lane and five shuffles; the in-kernel walk adds K / 4 values per lane and two shuffles
  (<= 130 adds at K = 512), so the factor 2.
* rowsums (producer): the output bits equal ops.gemm's; every slot and the sum over slots of each row are within
  (BN + nparts) u sum|h| of the fp64 sum of the output bits they cover (a slot is BN / 8 sequential adds per lane and two
  shuffles over BN / 2 columns), for sums of h and of h^2; nparts = 2 N / BN; slots >= nparts and rows >= M are not written.

A correct kernel stays below ratio 1 on any input, so a ratio above 1 is a bug, not a tolerance to widen.

2. Against the operation (``operation_ref64``): ref = LayerNorm64(x) W64^T + b on the ORIGINAL parameters (w, gamma, beta, b),
judged against the bound of the default path for the same call: the LayerNorm kernel's bound (layernorm_ref64) plus the
rounding of its output to bf16, propagated through |W|, plus the GEMM bound on that output.  Let rho = |mean| / sigma of a
row, z_k = (x_k - mu) r.  Beyond what the default path also pays, the fused paths add
  (a) the weight rounding bf16(gamma w): 2^-9 r sum_k |x_k - mu| |gamma_k w_k| = 2^-9 sum |z_k gamma_k w_k| -- CENTRED, only
      because colsum sums the rounded weights (``test_fold_layernorm_packing_is_exact``); the default path's LayerNorm
      output rounding is 2^-8 sum |z_k gamma_k w_k|, twice this;
  (b) + (c) the uncentred accumulation and mu colsum: (K + 2) 2^-22 r sum_k |x_k| |wf_k| <= (K + 2) 2^-22 (rho sum |wf_k| +
      sum |z_k wf_k|);
  (d) the statistics: lnfold / gemm_ln 2^-17 (rho + max|z|) |colsum| (small), lnparts the raw variance: a relative rstd
      error ~ 1.5 (nparts + 2) u rho^2.
Giving (b) + (c) half of the slack (a) leaves, 2^-10 sum |z gamma w| with m = sum |z gamma w| / sum |gamma w| ~ 0.8 for
Gaussian rows, bounds the range where the fused bound stays under the default one:
      R(K) = 0.8 * 2^12 / (K + 2):   R(320) = 10.2,  R(640) = 5.1,  R(1280) = 2.6
and (d) stays inside the other half there for both modes (the hand-over needs rho^2 < 2^14 / (1.5 (nparts + 2)), rho < 11.5
even at nparts = 80).  Rows with rho <= R (and exactly zero rows, rho = 0) must meet the default path's bound (ratio <= 1);
rows beyond R (the far ``offset`` rows, ``near-constant``) are checked by section 1 only, and their fused and default
errors are printed side by side.  ``test_synthetic_unet_layernorm_inputs`` prints the largest rho over every LayerNorm
input row of the synthetic small and full-width UNets (the oracle's ``layer_norm`` wrapped on the CPU) and requires it to
be inside R: that is a statement about these synthetic weights only; real checkpoint weights were not available.

3. Data families (functions of a torch.Generator, shared by the CPU self-test and the GPU cases):
  flat          : N(0, 1) rows, gamma 1 + N(0, 0.25), beta N(0, 0.5).
  row-scale     : rows scaled 2^-6, 1, 2^6 by m mod 3: statistics of a neighbouring row, of the thread's other row (m ^ 8)
                  or of the previous row tile (m - 128) are off by 2^6.
  offset        : row m has mean rho_m sigma_m, rho_m = 64 (m mod 17) / 16 from 0 to 64, sigma_m in [0.5, 2].
  near-constant : sigma = 2^-7 |mean| (a few bf16 ulp around the mean, mean in +-[1, 8]), every fifth row exactly constant.
  zero-rows     : flat with every fourth row exactly zero (r = eps^-1/2: the output is bf alone).
  frames        : per-frame bias2 (rows_per_frame not a multiple of 128), frames scaled 4^(n mod 3) and shifted by 3 n mod 5.
  wide-gate     : GEGLU gate rows of W x 4: gates over +-8.
``test_bound_rejects_injected_faults`` runs ``emulate_lnfold`` (a torch model of the epilogue arithmetic in the kernel's
fp32 order, with the three statistics sources) through the section 1 check: the correct model stays <= 1 on every family,
and each fault of ``FAULTS`` exceeds 1 on at least one.

Outputs go into the interior of sentinel-filled (NaN) buffers with a leading dimension larger than N, operands are
interior views of such buffers: a stray read turns an output into NaN, a stray write shows in the border.
"""
import contextlib
import ctypes
import math
import os

import pytest
import torch
import torch.nn.functional as F

from test_gemm_bounds_gpu import (_border_untouched, _bordered, _chunks, _f32, _in_nan, _INNER, _sentinel_buf,
                                  _SENTINEL32, bound_check, geglu_propagate, linear_ref64)
from test_norm_bounds_gpu import layernorm_ref64, row_stats_ref64

U = 2.0 ** -24
EPS = 1e-5
FAMILIES = ("flat", "row-scale", "offset", "near-constant", "zero-rows", "frames", "wide-gate")
R_M = 0.8                        # sum |z gamma w| / sum |gamma w| of Gaussian rows (section 2)
_WORST = {}                      # path -> (worst ratio, case)
_PARITY = []                     # rows of the fused-versus-default table


def R(K):
    """|mean| / sigma up to which a fused path keeps the default path's accuracy bound (module docstring, section 2)."""
    return R_M * 2.0 ** 12 / (K + 2)


def _g(x):
    return torch.tensor(float(x), dtype=torch.float64)


# ---------------------------------------------------------------------------------------------------------- references
def lnfold_ref64(A, wf, cs, bf, mu, r, dmu=None, dr=None, bias2=None, div=1, scale=1.0, residual=None, row0=0, geglu_bn=0):
    """(ref, bound without the output rounding) of the normalising epilogue for rows A [rows, K] (exact values) with the
    statistics (mu, r) [rows] known to within (dmu, dr) [rows] (None: exact).  geglu_bn: wf / cs / bf packed per column
    tile of that width (value half, gate half); the output has N / 2 columns."""
    K = A.shape[1]
    Ad, Wd = A.double(), wf.double()
    acc, P = Ad @ Wd.t(), Ad.abs() @ Wd.abs().t()
    mu, r = mu.double()[:, None], r.double()[:, None]
    c = cs.double()[None, :]
    mcs = mu * c
    t = acc - mcs
    dt = K * 2.0 ** -22 * P + 2.0 ** -22 * (P + mcs.abs())
    if dmu is not None:
        dt = dt + c.abs() * dmu.double()[:, None]
    z = r * t
    dz = r * dt
    if dr is not None:
        drr = dr.double()[:, None]
        dz = dz + torch.where(t.abs() + dt == 0, torch.zeros_like(dz), drr * (t.abs() + dt))
    b = bf.double()[None, :]
    if geglu_bn:
        rows, N = z.shape
        h = geglu_bn // 2
        split = lambda q: (q.reshape(rows, N // geglu_bn, 2, h)[:, :, 0].reshape(rows, -1),
                           q.reshape(rows, N // geglu_bn, 2, h)[:, :, 1].reshape(rows, -1))
        (zv, zg), (dzv, dzg), (bv, bg) = split(z), split(dz), split(b.expand(rows, N))
        V, G = zv + bv, zg + bg
        return geglu_propagate(V, G, dzv + 2.0 ** -22 * (zv.abs() + bv.abs()), dzg + 2.0 ** -22 * (zg.abs() + bg.abs()))
    lin, lin_abs = z + b, z.abs() + dz + b.abs()
    if bias2 is not None:
        idx = (row0 + torch.arange(A.shape[0], device=A.device)) // div
        b2 = bias2.reshape(-1, bias2.shape[-1])[idx].double()
        lin, lin_abs = lin + b2, lin_abs + b2.abs()
    s = _f32(scale)
    ref, ref_abs = s * lin, abs(s) * lin_abs
    if residual is not None:
        ref, ref_abs = ref + residual.double(), ref_abs + residual.double().abs()
    return ref, abs(s) * dz + 2.0 ** -20 * ref_abs


def lnfold_ref64_chunked(A, wf, cs, bf, st, **kw):
    """lnfold_ref64 over row chunks; st = (mu, r, dmu, dr) [rows] each (dmu / dr may be None)."""
    M, N = A.shape[0], wf.shape[0]
    ncol = N // 2 if kw.get("geglu_bn") else N
    ref = torch.empty((M, ncol), dtype=torch.float64, device=A.device)
    bnd = torch.empty_like(ref)
    kw = dict(kw)
    res = kw.pop("residual", None)
    for r0, r1 in _chunks(M, A.shape[1], 2 * N):
        sl = lambda v: None if v is None else v[r0:r1]
        ref[r0:r1], bnd[r0:r1] = lnfold_ref64(A[r0:r1], wf, cs, bf, *[sl(v) for v in st], residual=sl(res), row0=r0, **kw)
    return ref, bnd


def stats_exact(st):
    """(mu, r, None, None) of an fp32 [rows, 2] statistics array the kernel read."""
    return st[:, 0], st[:, 1], None, None


def parts_stats64(parts, nparts, K, eps=EPS):
    """(mu, r, d_mu, d_r) rebuilt in fp64 from the partial slots [>= nparts, rows, 2] (module docstring, lnparts)."""
    p = parts[:nparts].double()
    S1, S2, A1 = p[..., 0].sum(0), p[..., 1].sum(0), p[..., 0].abs().sum(0)
    mu, E2 = S1 / K, S2 / K
    v = torch.clamp(E2 - mu * mu, min=0)
    e = _f32(eps)
    dmu = nparts * U * A1 / K + 2 * U * mu.abs()
    dv = (nparts + 2) * U * E2 + 2 * mu.abs() * dmu + dmu * dmu + 2 * U * (E2 + mu * mu) + U * (v + e)
    x = dv / (v + e)
    rel = torch.where(x < 1, (1 - x.clamp(max=0.999999)).rsqrt() - 1, torch.full_like(x, math.inf)) + 2.0 ** -22
    r = (v + e).rsqrt()
    return mu, r, dmu, r * rel


def ln_stats64(x, eps=EPS):
    """(mu, r, d_mu, d_r) of the in-kernel two-pass statistics of gemm_ln: row_stats_ref64 with twice its bound."""
    ref, bnd = row_stats_ref64(x, eps)
    return ref[:, 0], ref[:, 1], 2 * bnd[:, 0], 2 * bnd[:, 1]


def operation_ref64(x, w, b, gamma, beta, eps=EPS, bias2=None, div=1, geglu=False):
    """(ref, default-path bound without the output rounding) of LayerNorm64(x) w^T + b (+ b2 | GEGLU) on the original
    parameters; w unpacked (GEGLU: value rows, then gate rows)."""
    M, K = x.shape
    N = w.shape[0]
    ref = torch.empty((M, N // 2 if geglu else N), dtype=torch.float64, device=x.device)
    bnd = torch.empty_like(ref)
    Wd, Wa = w.double(), w.double().abs()
    for r0, r1 in _chunks(M, K, 4 * N):
        n, ln_b = layernorm_ref64(x[r0:r1], gamma, beta, eps)
        dn = ln_b + 2.0 ** -8 * (n.abs() + ln_b)                 # the LayerNorm kernel's bound + its bf16 output rounding
        na = n.abs() + dn
        lin = n @ Wd.t() + b.double()
        P = na @ Wa.t()
        d = dn @ Wa.t() + K * 2.0 ** -22 * P                      # propagated through |W|, plus the GEMM's accumulation
        if geglu:
            h = N // 2
            dV = d[:, :h] + 2.0 ** -22 * (P[:, :h] + b[:h].double().abs())
            dG = d[:, h:] + 2.0 ** -22 * (P[:, h:] + b[h:].double().abs())
            ref[r0:r1], bnd[r0:r1] = geglu_propagate(lin[:, :h], lin[:, h:], dV, dG)
            continue
        ref_abs = P + b.double().abs()
        if bias2 is not None:
            b2 = bias2[(r0 + torch.arange(r1 - r0, device=x.device)) // div].double()
            lin, ref_abs = lin + b2, ref_abs + b2.abs()
        ref[r0:r1], bnd[r0:r1] = lin, d + 2.0 ** -20 * ref_abs
    return ref, bnd


def row_rho(x):
    """|mean| / sigma per row (fp64; 0 for an all-zero row, inf for a constant non-zero row)."""
    xd = x.double()
    mu = xd.mean(1)
    sd = ((xd - mu[:, None]) ** 2).mean(1).sqrt()
    rho = torch.where(sd > 0, mu.abs() / sd.clamp_min(1e-300), torch.where(mu == 0, torch.zeros_like(mu),
                                                                            torch.full_like(mu, math.inf)))
    return rho


# ------------------------------------------------------------------------------------------------------- data families
def lnf_inputs(fam, g, M, K, N, *, geglu=False, div=0):
    """bf16 x [M, K], bf16 w [N, K] (GEGLU: unpacked), fp32 bias [N], gamma [K], beta [K], bias2 [rows, N] or None."""
    dev = g.device
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    rows = torch.arange(M, device=dev)
    x = rn(M, K)
    if fam == "row-scale":
        x = x * torch.exp2(6.0 * ((rows % 3) - 1).float())[:, None]
    elif fam == "offset":
        rho = 64.0 * (rows % 17).float() / 16
        sig = torch.exp2(2 * torch.rand(M, device=dev, generator=g) - 1)
        sign = torch.where(torch.rand(M, device=dev, generator=g) < 0.5, -1.0, 1.0)
        x = (sign * rho * sig)[:, None] + sig[:, None] * x
    elif fam == "near-constant":
        mu = (1 + 7 * torch.rand(M, device=dev, generator=g)) * torch.where(torch.rand(M, device=dev, generator=g) < 0.5, -1.0, 1.0)
        x = mu[:, None] * (1 + 2.0 ** -7 * x)
        x[rows % 5 == 2] = mu[rows % 5 == 2, None].bfloat16().float()
    elif fam == "zero-rows":
        x[rows % 4 == 1] = 0
    elif fam == "frames":
        d = div or 100
        fr = (rows // d).float()
        x = x * (4.0 ** (fr % 3))[:, None] + (3.0 * (fr % 5))[:, None]
    w = rn(N, K) / math.sqrt(K)
    if geglu and fam == "wide-gate":
        w[N // 2:] *= 4
    gamma = 1 + 0.25 * rn(K)
    beta = 0.5 * rn(K)
    b = (0.5 * rn(N)).bfloat16().float()
    b2 = None
    if div:
        nb2 = (M - 1) // div + 1
        b2 = rn(nb2, N) * (4.0 ** (torch.arange(nb2, device=dev) % 3).float()[:, None] if fam == "frames" else 1.0)
    return x.bfloat16(), w.bfloat16(), b, gamma, beta, b2


def fold(w, b, gamma, beta, geglu=False, bn=0):
    """ops.fold_layernorm (CPU or GPU tensors); bn: the GEGLU tile width it packs at."""
    from vexpress_b200 import ops
    wf, cs, bf = ops.fold_layernorm(w, b, gamma, beta, geglu=geglu)
    return wf, cs, bf, (ops.geglu_block_n(w.shape[0]) if geglu else 0)


# ------------------------------------------------------------------------------------------------------------ emulation
FAULTS = ("row_prev", "row_next", "row_h8", "rstd_first", "colsum_unrounded", "sv_sg_swapped", "bias2_inside",
          "slot_dropped", "slot_twice", "eps_omitted", "eps_outside", "prev_tile", "residual_excluded")
# faults that only exist for one statistics source / epilogue kind
_FAULT_SOURCE = {"slot_dropped": "parts", "slot_twice": "parts", "residual_excluded": "parts", "prev_tile": "ln",
                 "eps_omitted": ("parts", "ln"), "eps_outside": ("parts", "ln")}


def producer_parts(h, bn):
    """The rowsums slots of a bf16 producer output h [M, N] at column tile bn: [2 N / bn, M, 2] fp32 (sum, sum of squares)
    over each half tile."""
    M, N = h.shape
    hf = h.float().reshape(M, 2 * N // bn, bn // 2)
    return torch.stack([hf.sum(2), (hf * hf).sum(2)], 2).permute(1, 0, 2).contiguous()


def _rstd32(var, eps, fault):
    e = torch.tensor(eps, dtype=torch.float32)
    if fault == "eps_omitted":
        return torch.rsqrt(var)
    if fault == "eps_outside":
        return torch.rsqrt(var) + e
    return torch.rsqrt(var + e)


def emulate_lnfold(A, wf, cs, bf, source, *, stats=None, parts=None, nparts=0, eps=EPS, bias2=None, div=1, scale=1.0,
                   residual=None, geglu_bn=0, fault=None):
    """Torch model of the LNF epilogue in the kernel's fp32 order.  source: 'stats' (the (mean, rstd) array ``stats``),
    'parts' (the producer slots, summed in slot order; variance E[x^2] - mean^2) or 'ln' (two-pass statistics of A)."""
    M, K = A.shape
    if source == "stats":
        mu, r = stats[:, 0].float(), stats[:, 1].float()
    elif source == "parts":
        n = nparts - 1 if fault == "slot_dropped" else nparts
        s1 = torch.zeros(M, dtype=torch.float32)
        s2 = torch.zeros(M, dtype=torch.float32)
        for j in range(n):
            s1, s2 = s1 + parts[j, :, 0], s2 + parts[j, :, 1]
        if fault == "slot_twice":
            s1, s2 = s1 + parts[0, :, 0], s2 + parts[0, :, 1]
        invK = torch.tensor(1.0 / K, dtype=torch.float32)
        mu = s1 * invK
        r = _rstd32(torch.clamp(s2 * invK - mu * mu, min=0), eps, fault)
    else:
        xf = A.float()
        mu = xf.sum(1) * torch.tensor(1.0 / K, dtype=torch.float32)
        d = xf - mu[:, None]
        r = _rstd32((d * d).sum(1) * torch.tensor(1.0 / K, dtype=torch.float32), eps, fault)
    rows = torch.arange(M)
    idx = {"row_prev": (rows - 1).clamp(min=0), "row_next": (rows + 1).clamp(max=M - 1),
           "row_h8": torch.where((rows ^ 8) < M, rows ^ 8, rows),
           "prev_tile": torch.where(rows >= 128, rows - 128, rows)}.get(fault)
    if idx is not None:
        mu, r = mu[idx], r[idx]
    acc = A.float() @ wf.float().t()
    if fault == "rstd_first":
        z = r[:, None] * acc - mu[:, None] * cs[None, :]
    else:
        t = acc - mu[:, None] * cs[None, :]
        if fault == "bias2_inside" and bias2 is not None:
            t = t + bias2[rows // div].float()
        z = r[:, None] * t
    if geglu_bn:
        h = geglu_bn // 2
        zt = (z + bf[None, :]).reshape(M, -1, 2, h)
        return (zt[:, :, 0] * F.gelu(zt[:, :, 1])).reshape(M, -1).bfloat16()
    y = z + bf[None, :]
    if bias2 is not None and fault != "bias2_inside":
        y = y + bias2[rows // div].float()
    y = y * _f32(scale)
    if residual is not None:
        y = y + residual.float()
    return y.bfloat16()


def _swap_halves(v, bn):
    """cs with the value and gate halves of every packed column tile exchanged (sv <-> sg)."""
    return v.reshape(-1, 2, bn // 2).flip(1).reshape(-1).contiguous()


def _cpu_case(fam, source, g):
    """-> (run(fault) -> out, ref, bnd, applies(fault)) for one family and statistics source on the CPU."""
    geglu = fam == "wide-gate"
    M, K, N = 300, 128, 256 if geglu else 128
    div = 100 if fam == "frames" else 0
    x, w, b, gamma, beta, b2 = lnf_inputs(fam, g, M, K, N, geglu=geglu, div=div)
    wf, cs, bf, gbn = fold(w, b, gamma, beta, geglu=geglu)
    cs_raw = (w.float() * gamma[None, :]).sum(1)
    if geglu:
        from vexpress_b200 import ops
        cs_raw = ops.pack_geglu(cs_raw[:, None], None)[0][:, 0].contiguous()
    res = (None if geglu else torch.randn(M, N, generator=g).bfloat16())
    kw = dict(bias2=b2, div=div or 1, scale=1.0 if geglu else 0.75, residual=res, geglu_bn=gbn)
    if geglu:
        kw.update(bias2=None, scale=1.0)
    A, parts, nparts, stats, parts_raw = x, None, 0, None, None
    if source == "parts":
        # the consumer's A is a producer's output h = bf16(a_p W_p^T + b_p + res_p); the family lives in res_p
        Kp = 64
        a_p = torch.randn(M, Kp, generator=g).bfloat16()
        w_p = (0.25 * torch.randn(K, Kp, generator=g) / math.sqrt(Kp)).bfloat16()
        pre = (a_p.float() @ w_p.float().t()).bfloat16().float()
        A = (pre + x.float()).bfloat16()
        parts = producer_parts(A, 64)
        nparts = parts.shape[0]
        parts_raw = producer_parts(pre.bfloat16(), 64)
        st = parts_stats64(parts, nparts, K)
    elif source == "stats":
        xf = x.float()
        mu = xf.mean(1)
        stats = torch.stack([mu, torch.rsqrt(((xf - mu[:, None]) ** 2).mean(1) + torch.tensor(EPS, dtype=torch.float32))], 1)
        st = stats_exact(stats)
    else:
        st = ln_stats64(x)
    ref, bnd = lnfold_ref64_chunked(A, wf, cs, bf, st, **kw)

    def run(fault):
        c = cs_raw if fault == "colsum_unrounded" else _swap_halves(cs, gbn) if fault == "sv_sg_swapped" else cs
        p = parts_raw if fault == "residual_excluded" else parts
        return emulate_lnfold(A, wf, c, bf, source, stats=stats, parts=p, nparts=nparts, fault=fault, **kw)

    def applies(fault):
        src = _FAULT_SOURCE.get(fault)
        if src and source not in ((src,) if isinstance(src, str) else src):
            return False
        if fault == "sv_sg_swapped":
            return geglu
        if fault == "bias2_inside":
            return b2 is not None and not geglu
        return True
    return run, ref, bnd, applies


def test_bound_rejects_injected_faults():
    """The faithful model is <= 1 on every family and source; every fault exceeds 1 on at least one family (table)."""
    table = {f: {} for f in FAULTS}
    for i, fam in enumerate(FAMILIES):
        for source in ("stats", "parts", "ln"):
            run, ref, bnd, applies = _cpu_case(fam, source, torch.Generator().manual_seed(300 + 7 * i))
            worst, rel, where = bound_check(run(None), ref, bnd)
            print(f"faithful model {source:5s} {fam:13s}: worst ratio {worst:.3f}")
            assert worst <= 1, (fam, source, where)
            for fault in FAULTS:
                if applies(fault):
                    worst, _, _ = bound_check(run(fault), ref, bnd)
                    table[fault][(fam, source)] = max(worst, table[fault].get((fam, source), 0.0))
    print(f"\n{'fault':18s} " + " ".join(f"{f[:11]:>11s}" for f in FAMILIES) + "   (worst ratio over the statistics sources)")
    for fault, hits in table.items():
        cells = []
        for fam in FAMILIES:
            vals = [v for (f, _), v in hits.items() if f == fam]
            cells.append(f"{max(vals):11.3g}" if vals else f"{'-':>11s}")
        print(f"{fault:18s} " + " ".join(cells))
    for fault, hits in table.items():
        n = sum(1 for v in hits.values() if v > 1)
        assert n >= 1, f"{fault} passes every family"


def test_cpu_references_agree():
    """lnfold_ref64 (with the exact fp64 statistics) and operation_ref64 against F.layer_norm / @ in float64: the fold
    algebra and the GEGLU packing of the references are themselves right."""
    g = torch.Generator().manual_seed(11)
    M, K, N = 40, 64, 128
    x, w, b, gamma, beta, b2 = lnf_inputs("frames", g, M, K, N, div=7)
    want = F.layer_norm(x.double(), (K,), gamma.double(), beta.double(), _f32(EPS)) @ w.double().t() + b.double()
    want = want + b2.double()[torch.arange(M) // 7]
    ref, _ = operation_ref64(x, w, b, gamma, beta, bias2=b2, div=7)
    torch.testing.assert_close(ref, want)
    # the fold on fp64 weights (no rounding) is the same operation
    wf64 = w.double() * gamma.double()[None, :]
    xd = x.double()
    mu = xd.mean(1)
    r = (((xd - mu[:, None]) ** 2).mean(1) + _f32(EPS)).rsqrt()
    ref, _ = lnfold_ref64(x, wf64, wf64.sum(1), w.double() @ beta.double() + b.double(), mu, r, bias2=b2, div=7)
    torch.testing.assert_close(ref, want)
    # GEGLU: packed fold, unpacked operation
    x, w, b, gamma, beta, _ = lnf_inputs("wide-gate", g, M, K, 256, geglu=True)
    want = F.layer_norm(x.double(), (K,), gamma.double(), beta.double(), _f32(EPS)) @ w.double().t() + b.double()
    want = want[:, :128] * F.gelu(want[:, 128:])
    torch.testing.assert_close(operation_ref64(x, w, b, gamma, beta, geglu=True)[0], want)
    from vexpress_b200 import ops
    wf64 = w.double() * gamma.double()[None, :]
    wp, bp, bn = ops.pack_geglu(wf64, w.double() @ beta.double() + b.double())
    xd = x.double()
    mu = xd.mean(1)
    r = (((xd - mu[:, None]) ** 2).mean(1) + _f32(EPS)).rsqrt()
    torch.testing.assert_close(lnfold_ref64(x, wp, wp.sum(1), bp, mu, r, geglu_bn=bn)[0], want)


def test_fold_layernorm_packing_is_exact():
    """ops.fold_layernorm: colsum is the fp32 sum of the RETURNED (rounded) wf, bf = w beta + b, the GEGLU order is
    pack_geglu's; and r (A wf^T - mu colsum) + bf in fp64 equals LayerNorm64(A) (gamma w)^T + w beta + b up to the centred
    weight-rounding term 2^-9 r sum |a_k - mu| |gamma_k w_k| (plus the fp32 roundings of colsum and bf), on rows with
    |mean| / sigma up to 64.  A colsum of the unrounded gamma w leaves an uncentred residue and fails the same check."""
    from vexpress_b200 import ops
    g = torch.Generator().manual_seed(12)
    M, K, N = 300, 320, 192
    x, w, b, gamma, beta, _ = lnf_inputs("offset", g, M, K, N)
    wf, cs, bf = ops.fold_layernorm(w, b, gamma, beta)
    assert wf.dtype == torch.bfloat16 and cs.dtype == torch.float32 and bf.dtype == torch.float32
    assert torch.equal(wf, (w.float() * gamma[None, :]).bfloat16())
    assert torch.equal(cs, wf.float().sum(1))
    wfd = wf.double()
    assert ((cs.double() - wfd.sum(1)).abs() <= K * U * wfd.abs().sum(1)).all()
    bf64 = w.double() @ beta.double() + b.double()
    bf_tol = K * U * (w.double().abs() @ beta.double().abs()) + U * b.double().abs()
    assert ((bf.double() - bf64).abs() <= bf_tol).all()
    wg, cg, bg = ops.fold_layernorm(w, b, gamma, beta, geglu=True)
    pw, pb, _ = ops.pack_geglu(wf, bf)
    assert torch.equal(wg, pw) and torch.equal(bg, pb) and torch.equal(cg, wg.float().sum(1))
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    r = (((xd - mu) ** 2).mean(1, keepdim=True) + _f32(EPS)).rsqrt()
    gw = w.double() * gamma.double()[None, :]
    want = (xd - mu) * r @ gw.t() + bf64
    tol = (2.0 ** -9 * r * ((xd - mu).abs() @ gw.abs().t())
           + r * mu.abs() * (K * U * wfd.abs().sum(1))[None, :] + bf_tol[None, :] + 1e-12 * want.abs())
    got = r * (xd @ wfd.t() - mu * cs.double()[None, :]) + bf.double()
    ratio = ((got - want).abs() / tol).max().item()
    cs_raw = gw.float().sum(1).double()
    bad = r * (xd @ wfd.t() - mu * cs_raw[None, :]) + bf.double()
    bad_ratio = ((bad - want).abs() / tol).max().item()
    print(f"fold algebra: worst ratio {ratio:.3f} with colsum of the rounded weights, {bad_ratio:.3g} with the unrounded")
    assert ratio <= 1 and bad_ratio > 1


def test_synthetic_unet_layernorm_inputs():
    """Largest |mean| / sigma over every LayerNorm input row of the synthetic small (K = 64..256) and full-width
    (K = 320..1280) UNets, recorded by wrapping the oracle's layer_norm: it must lie inside R(K) of the LayerNorm's width.
    Synthetic weights only: real checkpoint weights may put rows elsewhere."""
    from oracle import vx_oracle as O
    seen = {}
    orig = O.layer_norm

    def rec(sd, p, x):
        rho = row_rho(x.reshape(-1, x.shape[-1]))
        K = x.shape[-1]
        seen[K] = max(seen.get(K, 0.0), float(rho[torch.isfinite(rho)].max()))
        return orig(sd, p, x)
    O.layer_norm = rec
    try:
        for name, cfg, L, hw in (("small", O.small_cfg(), 4, 16), ("full-width", O.DEFAULT_CFG, 2, 16)):
            seen.clear()
            sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
            lat, kps, audio, banks = O.synth_inputs(cfg, L, hw, hw, True, 42)
            with torch.no_grad():
                O.unet_forward(sd, cfg, lat.repeat(2, 1, 1, 1, 1), 499, audio.reshape(-1, 5, cfg["cross_attention_dim"]),
                               kps, banks, 0.95, 3.0)
            print(f"synthetic {name} UNet: largest |mean| / sigma of a LayerNorm input row, by width: "
                  + ", ".join(f"K {k}: {v:.3f} (R {R(k):.1f})" for k, v in sorted(seen.items())))
            for k, v in seen.items():
                assert v <= R(k), (name, k, v)
            del sd
    finally:
        O.layer_norm = orig


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for path, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {path:16s} {worst:.3f}  ({case})")
    if _PARITY:
        print(f"\n{'fused vs default':44s} {'rho range':>13s} {'rows':>6s} {'fused/bnd':>10s} {'deflt/bnd':>10s} "
              f"{'fused rel':>10s} {'deflt rel':>10s}")
        for row in _PARITY:
            print("{:44s} {:>13s} {:6d} {:10.3f} {:10.3f} {:10.2e} {:10.2e}".format(*row))


@pytest.fixture
def force_bn():
    """force_bn(bn) sets VX_GEMM_BN (0: the dispatcher's choice) and makes the library re-read it."""
    from vexpress_b200 import _ffi
    before = os.environ.get("VX_GEMM_BN")

    def switch(bn):
        if bn:
            os.environ["VX_GEMM_BN"] = str(bn)
        else:
            os.environ.pop("VX_GEMM_BN", None)
        _ffi.lib().vx_gemm_reload_env()
    yield switch
    if before is None:
        os.environ.pop("VX_GEMM_BN", None)
    else:
        os.environ["VX_GEMM_BN"] = before
    _ffi.lib().vx_gemm_reload_env()


def _seed(*xs):
    s = 0
    for v in xs:
        s = (s * 1000003 + sum(map(ord, str(v)))) % (1 << 31)
    return s


def _record(path, case, fam, out, ref, bnd, border=""):
    torch.cuda.synchronize()
    worst, rel, where = bound_check(out, ref, bnd)
    print(f"{path:8s} {case} {fam:13s}: worst ratio {worst:.3f}, rel {rel:.2e}")
    if worst > _WORST.get(path, (-1.0, ""))[0]:
        _WORST[path] = (worst, f"{case} {fam}")
    bad = []
    if not worst <= 1:
        bad.append(f"bound exceeded, {where}")
    if torch.isnan(out.float()).any():
        bad.append("NaN left in the output")
    if border:
        bad.append(border)
    return f"{path} {case} {fam}: " + "; ".join(bad) if bad else ""


def _rowsums(ops, h_in, w, b, res, M, N):
    """vx_gemm_rowsums_bf16 into sentinel-filled out / parts buffers (parts rows M.. and slots nparts.. must stay
    untouched) -> (out view, out buffer, parts buffer [cap, M + 5, 2], nparts)."""
    from vexpress_b200 import _ffi
    from vexpress_b200._ffi import c_float, c_int, c_ll, check, ptr, stream_ptr
    obuf, out = _bordered(M, N)
    cap = ops.rowsum_slots(N)
    pbuf = _sentinel_buf((cap, M + 5, 2), torch.float32)
    nparts = c_int(0)
    check(_ffi.lib().vx_gemm_rowsums_bf16(
        ptr(h_in), c_ll(h_in.stride(0)), c_int(h_in.shape[1]), ptr(None), c_ll(0), c_int(0), ptr(w), c_ll(w.stride(0)),
        c_int(M), c_int(N), ptr(b), ptr(None), c_int(1), c_float(1.0), ptr(res), c_ll(0 if res is None else res.stride(0)),
        ptr(out), c_ll(out.stride(0)), c_int(0), ptr(pbuf), c_ll(M + 5), c_int(cap), ctypes.byref(nparts), stream_ptr()),
        "vx_gemm_rowsums_bf16")
    return out, obuf, pbuf, nparts.value


def _check_rowsums(ops, h, pbuf, nparts, M, N, twin):
    """The producer checks of the module docstring -> list of failure messages."""
    bad = []
    if not torch.equal(h, twin):
        bad.append("output bits differ from ops.gemm")
    bn = 2 * N // nparts
    if nparts * bn != 2 * N or bn not in (32, 64, 96, 128, 160, 192, 256):
        bad.append(f"nparts {nparts} is not 2 N / BN for a valid BN")
    bits = pbuf.view(torch.int32)
    if (bits[nparts:] != _SENTINEL32).any() or (bits[:, M:] != _SENTINEL32).any():
        bad.append("slots >= nparts or rows >= M written")
    hd = h.double()
    p = pbuf[:nparts, :M].double()
    cols = hd.reshape(M, nparts, bn // 2)
    for k, v in ((0, cols), (1, cols * cols)):
        tol = (bn + nparts) * U * v.abs().sum(2)
        if not ((p[..., k].t() - v.sum(2)).abs() <= tol).all():
            bad.append(f"a slot's {'sum' if k == 0 else 'sum of squares'} is off")
        tot = (p[..., k].sum(0) - v.sum((1, 2))).abs()
        if not (tot <= (bn + nparts) * U * v.abs().sum((1, 2))).all():
            bad.append(f"the row {'sums' if k == 0 else 'sums of squares'} are off")
    return bad


@contextlib.contextmanager
def _dispatcher_bn():
    """The producer GEMM (K output columns) at the dispatcher's column tile even while VX_GEMM_BN forces the consumer's."""
    from vexpress_b200 import _ffi
    before = os.environ.pop("VX_GEMM_BN", None)
    _ffi.lib().vx_gemm_reload_env()
    try:
        yield
    finally:
        if before is not None:
            os.environ["VX_GEMM_BN"] = before
        _ffi.lib().vx_gemm_reload_env()


def _run_paths(ops, paths, fam, M, K, N, *, geglu=False, div=0, residual=False, scale=1.0, tag="", again=False,
               parity=False):
    """One data set of family ``fam`` through each path in ``paths`` (section 1 check; section 2 when ``parity``) ->
    list of failure messages."""
    g = torch.Generator(device="cuda").manual_seed(_seed(fam, M, K, N, geglu, div))
    x, w, b, gamma, beta, b2 = lnf_inputs(fam, g, M, K, N, geglu=geglu, div=div)
    wf, cs, bf, gbn = fold(w, b, gamma, beta, geglu=geglu)
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16() if residual and not geglu else None
    case = f"M {M} K {K} N {N}{' geglu' if geglu else ''}{' div %d' % div if div else ''}{' res' if res is not None else ''}{tag}"
    kw = dict(bias2=b2, bias2_div=div or 1, scale=scale, residual=None if res is None else _in_nan(res))
    if geglu:
        kw = {}
    rkw = dict(bias2=b2, div=div or 1, scale=scale, residual=res, geglu_bn=gbn)
    bad = []
    for path in paths:
        A = x
        if path == "lnparts":
            # the consumer's input is a producer's output h = bf16(a_p W_p^T + b_p + x): the residual x carries the family,
            # the product and bias are 2^-12 small so that near-constant and zero rows stay what they are
            Kp = 64
            a_p = torch.randn(M, Kp, device="cuda", generator=g)
            a_p[x.float().abs().amax(1) == 0] = 0
            a_p = a_p.bfloat16()
            w_p = (2.0 ** -12 * torch.randn(K, Kp, device="cuda", generator=g) / math.sqrt(Kp)).bfloat16()
            b_p = None if fam == "zero-rows" else (2.0 ** -12 * torch.randn(K, device="cuda", generator=g)).bfloat16().float()
            with _dispatcher_bn():
                h, hbuf, pbuf, nparts = _rowsums(ops, _in_nan(a_p), _in_nan(w_p), b_p, _in_nan(x), M, K)
                twin = ops.gemm(a_p, w_p, b_p, residual=x)
            msgs = _check_rowsums(ops, h, pbuf, nparts, M, K, twin)
            border = _border_untouched(hbuf, _INNER)
            bad += [f"rowsums {case} {fam}: {m}" for m in msgs + ([border] if border else [])]
            A = h.clone()
            parts = pbuf[:, :M].contiguous()
            st = parts_stats64(parts, nparts, K)
            run = lambda o: ops.gemm_lnparts(_in_nan(A), _in_nan(wf), parts, nparts, cs, bf, EPS, out=o, geglu=geglu, **kw)
        elif path == "lnfold":
            stats = ops.row_stats(_in_nan(x))
            st = stats_exact(stats)
            run = lambda o: ops.gemm_lnfold(_in_nan(A), _in_nan(wf), stats, cs, bf, out=o, geglu=geglu, **kw)
        else:
            st = ln_stats64(x)
            run = lambda o: ops.gemm_ln(_in_nan(A), _in_nan(wf), cs, bf, EPS, out=o, geglu=geglu, **kw)
        obuf, out = _bordered(M, N // 2 if geglu else N)
        run(out)
        ref, bnd = lnfold_ref64_chunked(A, wf, cs, bf, st, **rkw)
        bad.append(_record(path, case, fam, out, ref, bnd, _border_untouched(obuf, _INNER)))
        if again:
            first = out.clone()
            torch.empty(1 << 22, device="cuda").normal_()
            run(out)
            torch.cuda.synchronize()
            if not torch.equal(out, first):
                bad.append(f"{path} {case} {fam}: two runs differ")
        if parity:
            bad.append(_parity(ops, path, case, fam, A, w, b, gamma, beta, b2, div, geglu, out))
    return [m for m in bad if m]


def _parity(ops, path, case, fam, A, w, b, gamma, beta, b2, div, geglu, out):
    """Section 2: the fused output against LayerNorm64(A) W^T + b under the default path's bound, rows with rho <= R(K)
    asserted, every rho range printed with the default path's own numbers beside it."""
    if b2 is not None or residual_in(case):
        return ""
    M, K = A.shape
    ref, bnd = operation_ref64(A, w, b, gamma, beta, geglu=geglu)
    if geglu:
        wg, bg, _ = ops.pack_geglu(w, b)
        dflt = ops.gemm(ops.layernorm(A, gamma, beta, EPS), wg, bg, geglu=True)
    else:
        dflt = ops.gemm(ops.layernorm(A, gamma, beta, EPS), w, b)
    torch.cuda.synchronize()
    tot = bnd + 2.0 ** -8 * ref.abs()
    rf = ((out.double() - ref).abs() / tot).nan_to_num(nan=math.inf).amax(1)
    rd = ((dflt.double() - ref).abs() / tot).nan_to_num(nan=math.inf).amax(1)
    rho = row_rho(A)
    msg = ""
    edges = [(0, R(K)), (R(K), 2 * R(K)), (2 * R(K), 16.0), (16.0, 64.5), (64.5, math.inf)]
    for lo, hi in edges:
        sel = (rho <= hi) & ((rho > lo) if lo > 0 else torch.ones_like(rho, dtype=torch.bool))
        if not sel.any():
            continue
        e = lambda o: float((o.double()[sel] - ref[sel]).norm() / ref[sel].norm().clamp_min(1e-30))
        _PARITY.append((f"{path} {case} {fam}", f"{lo:.3g}-{hi:.3g}", int(sel.sum()), float(rf[sel].max()),
                        float(rd[sel].max()), e(out), e(dflt)))
        if hi <= R(K) and not float(rf[sel].max()) <= 1:
            msg = (f"{path} {case} {fam}: rows with |mean|/sigma <= R({K}) = {R(K):.2f} exceed the default path's bound "
                   f"(ratio {float(rf[sel].max()):.3f})")
    return msg


def residual_in(case):
    return case.endswith(" res") or " res " in case


ALL_PATHS = ("lnfold", "lnparts", "gemm_ln")


# ---- ragged M: every family through the three paths; run-to-run identity once per path
@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 7, 127, 128, 129, 300, 128 * 133 + 1])
def test_ragged_rows_within_bound(ops, M):
    bad = []
    for fam in FAMILIES:
        geglu = fam == "wide-gate"
        bad += _run_paths(ops, ALL_PATHS, fam, M, 320, 384 if geglu else 320, geglu=geglu,
                          div=100 if fam == "frames" else 0, residual=fam == "flat", scale=0.75 if fam == "flat" else 1.0,
                          again=M == 300 and fam == "row-scale")
    assert not bad, "\n".join(bad)


# ---- every column tile width the dispatcher can pick, and bias2 with rows_per_frame not a multiple of 128
@pytest.mark.gpu
@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 256])
def test_every_block_n_within_bound(ops, force_bn, bn):
    force_bn(bn)
    bad = []
    for fam in ("row-scale", "frames", "offset"):
        bad += _run_paths(ops, ALL_PATHS, fam, 1000, 320, 3840, div=100 if fam == "frames" else 0, tag=f" bn {bn}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [192, 384, 2560])
def test_geglu_tile_widths_within_bound(ops, N):
    """The GEGLU packings at tiles 64, 128 and 256 (value / gate colsums sv, sg per tile)."""
    bad = []
    for fam in ("wide-gate", "row-scale", "offset"):
        bad += _run_paths(ops, ALL_PATHS, fam, 777, 320, N, geglu=True)
    assert not bad, "\n".join(bad)


# ---- the engine's shapes at 512 x 512 (rows = both CFG halves x f frames x the level's pixels), section 1 and 2
ENGINE = [(320, 4096), (640, 1024), (1280, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("f", [16, 24])
@pytest.mark.parametrize("kind", ["qkv", "to_q", "geglu"])
@pytest.mark.parametrize("K,HW", ENGINE)
def test_engine_shapes_within_bound(ops, K, HW, kind, f):
    N = {"qkv": 3 * K, "to_q": K, "geglu": 8 * K}[kind]
    paths = ALL_PATHS if K <= 512 else ALL_PATHS[:2]
    M = 2 * f * HW
    bad = []
    for fam in ("flat", "offset"):
        bad += _run_paths(ops, paths, fam, M, K, N, geglu=kind == "geglu", tag=f" f {f}", parity=True)
    assert not bad, "\n".join(bad)


# ---- section 2 on every family at the three widths
@pytest.mark.gpu
@pytest.mark.parametrize("K", [320, 640, 1280])
def test_parity_with_default_path(ops, K):
    bad = []
    paths = ALL_PATHS if K <= 512 else ALL_PATHS[:2]
    for fam in FAMILIES:
        if fam == "frames":
            continue
        geglu = fam == "wide-gate"
        bad += _run_paths(ops, paths, fam, 3000, K, 2 * K if geglu else K, geglu=geglu, parity=True)
    assert not bad, "\n".join(bad)


# ---- the UNet blocks under the two modes (tests/test_blocks_gpu.py's cases, criterion and thresholds unchanged)
MODES = {"fold": {"VX_LN_FOLD": "1", "VX_LN_FUSE": "0"}, "fuse": {"VX_LN_FOLD": "0", "VX_LN_FUSE": "1"}}


@pytest.fixture(scope="module")
def small_unet():
    from vexpress_b200 import _ffi
    from test_blocks_gpu import CFG, _unet, small_sd
    _ffi.require_sm90()
    return _unet(CFG, small_sd())


@pytest.fixture(scope="module")
def full_unet():
    from test_blocks_gpu import FULL_LEVELS, _full_keys, _unet
    from oracle import vx_oracle as O
    sd = _full_keys(tuple(p + "." for p, _ in FULL_LEVELS.values()))
    return sd, _unet(O.DEFAULT_CFG, sd, full=True)


def _in_mode(model, mode, body):
    """Run body() with the engine built under ``mode``; the engine is rebuilt in the default mode afterwards."""
    try:
        with pytest.MonkeyPatch.context() as mp:
            for k, v in MODES[mode].items():
                mp.setenv(k, v)
            model._engine = None
            out = body()
            eng = model.engine()
            assert (eng.ln_fold, eng.ln_fuse) == (mode == "fold", mode == "fuse")
            return out
    finally:
        model._engine = None


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("branch", ["attn1", "attn1_5", "attn2", "ff"])
@pytest.mark.parametrize("level", [0, 1, 2])
def test_spatial_branch_under_mode(small_unet, level, branch, mode):
    from test_blocks_gpu import FORMS, SPATIAL_LEVELS, _spatial_sweep, small_sd
    p, H = SPATIAL_LEVELS[level]
    _in_mode(small_unet, mode, lambda: _spatial_sweep(small_unet, small_sd(), p, H, branch, list(FORMS), (4,),
                                                      f"{mode} L{level}"))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("branch", ["attn1", "attn1_5", "attn2", "ff"])
@pytest.mark.parametrize("hd", [40, 80, 160])
def test_spatial_fullwidth_branch_under_mode(full_unet, hd, branch, mode):
    from test_blocks_gpu import FULL_LEVELS, _spatial_sweep
    sd, model = full_unet
    p, H = FULL_LEVELS[hd]
    _in_mode(model, mode, lambda: _spatial_sweep(model, sd, p, H, branch, ["uncond", "n2"], (4,), f"{mode} hd{hd}"))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("f", [1, 2, 16, 17, 24, 32])
@pytest.mark.parametrize("branch", ["attn0", "attn1", "ff"])
def test_motion_branch_under_mode(small_unet, branch, f, mode):
    """The motion module's positional encoding enters the fused paths as a per-frame bias2 (pe W^T, rows_per_frame = HW):
    test_blocks_gpu's catalogue shows its criterion rejects pe rows shifted by one frame (fault / threshold 16x)."""
    from test_blocks_gpu import (MIN_SHARE, MOTION_BLOCK, MOTION_BRANCHES, MOTION_GAIN, _load, _sub, isolate, judge,
                                 motion_case, run_motion, small_sd)
    sd = small_sd()
    p = MOTION_BLOCK

    def body():
        _load(small_unet, isolate(_sub(sd, p + "."), p + ".temporal_transformer.transformer_blocks.0", MOTION_BRANCHES,
                                  branch, MOTION_GAIN.get(branch, 1.0)))
        bad = []
        for bn in (1, 2, 4):
            c = motion_case(sd, p, branch, bn, f)
            assert c["share"] >= MIN_SHARE, (branch, f, bn, c["share"])
            bad.append(judge(f"motion {mode} {branch} f={f} bn={bn}", run_motion(small_unet, c), c))
        return [m for m in bad if m]
    bad = _in_mode(small_unet, mode, body)
    assert not bad, "\n".join(bad)
