"""GroupNorm (+SiLU, over [x1 | x2]), LayerNorm (+PE), row statistics, GEGLU, row softmax, the timestep embedding and the
skinny time-embedding linear against an fp64 reference of exactly the bf16 / fp32 values the kernel reads, element by
element, under an error bound a correct kernel cannot exceed (the counterpart of tests/test_gemm_bounds_gpu.py).

u = 2^-24 is the fp32 unit roundoff.  Every bf16 output adds 2^-8 |ref| (its one rounding, ``bound_check``); the other
terms bound what the kernel's fp32 arithmetic may add before it.

GroupNorm, per frame and group of N = HW cpg values x with mean mu, variance var (population), rstd = (var + eps)^-1/2,
z = (x - mu) rstd, y = z gamma + beta, out = y or silu(y):

    |out - ref| <= s'(y) D + e_act(y),   D = |gamma| (|z| d_rstd + rstd d_mean) + 2^-23 ((|x| + 2 |mu|) rstd |gamma| + |beta| + |y|)

* the statistics.  The kernels sum x - p in fp32, p = one value of the group (the pivot): each thread adds its pixels in
  sequence, a thread per group then adds the R pixel lanes x cpg channels, and the S (or cluster) partials merge by Chan's
  formula; ``n_add`` (``_gn_adds``) counts the fp32 adds on the longest of these paths.  A sum of n_add adds is off by at
  most n_add u sum |addend|, and sum (x - p)^2 = N (var + (mu - p)^2) <= N var (1 + k2), k2 = max (x - mu)^2 / var, the
  group's own spread.  So M2 = sum (x-p)^2 - (sum (x-p))^2 / N is off by (3 n_add + 8) u N var (1 + k2), and
      d_var  = (3 n_add + 8) u (1 + k2)                 (relative)
      d_rstd = (d_var var / (var + eps) + 2 u) / 2 + 4 u (rsqrtf: 2 ulp)
      d_mean = (2 n_add + 4) u max|x - mu| + u |mu|     (absolute: the shifted mean, and pivot + mean in fp32)
  Neither carries a (mu / std)^2 factor: that is what sums of x and x^2 without a shift would need (their M2 cancels to
  a relative u (mu / std)^2), and the ``offset`` family exists to show it.
* the apply: scale = rstd gamma, shift = beta - mean scale, y = fma(x, scale, shift): four roundings of values no larger
  than |x| rstd |gamma|, |mu| rstd |gamma|, |beta| and |y|, counted twice.
* SiLU: s'(y) = min(1.1, |silu'(y)| + D / 2) bounds |silu'| on [y - D, y + D] (|silu''| <= 1/2, |silu'| < 1.1).  The
  GroupNorm kernels compute 0.5 y (1 + tanh.approx(y / 2)): tanh.approx is within a relative 2^-11 of tanh (PTX ISA;
  2^-10.9 here), so e_act(y) = 2^-11.9 |y tanh(y / 2)| + 2^-22 |silu(y)|.  That term is stated, not hidden: below
  y = -4 it exceeds the bf16 rounding of silu(y) (at y = -8 it allows most of |silu(y)|); y / (1 + __expf(-y)) would be
  accurate to a few 2^-23 but took up to 1.38x the kernel time (tools/norm_ab_h100.txt).  A sigmoid of the unhalved argument,
  0.5 + 0.5 tanh(y), still fails the bound.  No SiLU: s' = 1, e_act = 0.
  The skinny linear's SiLU is y / (1 + __expf(-y)): e_act(y) = (5 + 1.2 |y|) 2^-23 |silu(y)| + 2^-126 (__expf within
  2 + 1.173 |y| ulp, one rounding for 1 + e and the division; below y = -80 the whole |silu(y)| < 2^-108).

LayerNorm of a row of C values (+ pe[(row // rows_per_frame) % pe_frames]):
    |out - ref| <= 2^-17 rstd |gamma| max|x_row| + 2^-18 |z gamma| + 2^-21 (|beta| + |pe|)
  The fp32 mean is a sum of <= 69 adds (64 values per lane in the one-warp-per-row kernel, then five shuffles), so it
  is off by < 2^-17.8 max|x_row|, which x - mean carries amplified by rstd (near-constant rows); the two-pass variance and
  rsqrtf give rstd to < 2^-18.5 relative; the products and the adds of beta and pe one u each.  This is the fp32 term of
  tests/test_fp8_gpu.py with the worst-case add count made explicit and the apply roundings split by operand.
Row statistics (fp32 out, no output rounding): the same mean term, 2^-17 max|x_row|, and 2^-18 rstd.
GEGLU out = h gelu(g), gelu(g) = g / 2 (1 + erff(g / sqrt 2)):  0.5 |h g| (2^-22 + 2^-23 |g|) + 2^-22 |ref|  (erff
  within 2 ulp, the argument's two roundings through erf' <= 1.13, 1 + erf, and three products).  A tanh-GELU is 10 %
  off around g = -3, where gelu is tiny: the bound rejects it.
Row softmax p = e^(x - m) / sum e^(x - m), t = x - m <= 0:
    |out - ref| <= p ((2 + 1.2 |t|) 2^-23 + u |t| + E + (n / 256 + 16) u + 2 u) + 2^-126
  __expf of t is within 2 + 1.173 |t| ulp and t itself carries u |t|, so the error grows with the distance from the row
  maximum; E = sum_j p_j (2 + 1.2 |t_j|) 2^-23 is what those errors do to the sum, whose n / 256 + 16 sequential adds
  (four per float4, a 32-lane shuffle tree, eight warps) add the next term; the reciprocal and the product one u each.
  Values below the fp32 normal range may be flushed: 2^-126 absolute.
Timestep embedding [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(10000) i / half), bf16-rounded: the reference is the same
  formula in torch at fp32 (what the reference model computes before its cast to bf16), compared before that cast:
  2^-8 |ref| (the cast) + 2^-19 |t f_i| + 2^-21 (two fp32 evaluations of the argument, a few ulp of exp / log each,
  and of cos / sin).
Skinny linear y = act_out(sum_k act_in(x_k) w_k + b), fp32 out: (K / 32 + 8) u sum |a_k w_k| for the lane-sequential
  sums and the shuffle tree, sum |w_k| e_act(x_k) for a SiLU on the input, u |b|, and s' / e_act as above on the output.

A correct kernel stays below the bound on any input, so a ratio above 1 is a bug, not a tolerance to widen.  Every case
also keeps the global criterion ||out - ref|| < 5e-3 ||ref||.

Data families (functions of a torch.Generator, shared by the CPU self-test and the GPU cases):
  flat           : N(0, 1); gamma 1 + N(0, 0.5), beta N(0, 0.5), so that y crosses zero where |z gamma| ~ 1.
  offset         : every group a bf16-exact mu + k ulp(mu) with mu / std from ~10 to ~250; group 0 of each frame near
                   constant (1000, 1 % of the pixels +-1 ulp), group 1 all constant (output = beta), group 2
                   bf16(1000 + 4 N(0, 1)).
  channel-spread : channels scaled 2^+6 or 2^-6 at random: a channel dropped from, or added to, a group's statistics shows.
  frames         : frame n scaled by 4^(n mod 3) and shifted by 3 (n mod 3), group g shifted by g mod 4: statistics of
                   the neighbouring frame or group show.
  tiny-var       : var = k^2 eps with k in [0.3, 3] per group, at eps 1e-5 and 1e-6: a swapped eps shows.
  silu-tail      : gamma in [2, 5], beta in [-12, -4]: pre-activations down to -30.
  pe             : (LayerNorm) rows with offsets N(0, 2), a PE table of fewer frames than the rows have, rows_per_frame
                   13 (no multiple of the rows a warp handles).
  gate           : (GEGLU) gates N(0, 3): the erf tails are used.
``test_norm_bound_rejects_injected_faults`` runs a torch model of each kernel's arithmetic (fp32 statistics of x - pivot per
pixel chunk, Chan merge in the kernel's lane / shuffle order, fp32 apply, bf16 output) with injectable faults through the
same check: the evidence that the GPU cases would catch those faults in the kernels.

Inputs are interior views of NaN-filled buffers (leading dimensions > C, multiples of 8; x1 and x2 in different buffers),
outputs go into the interior of sentinel-filled buffers: a stray read turns an output into NaN, a stray write shows in
the border.  Every GroupNorm path is called through its own entry point and must return 0 (the cluster and one-launch
entries return 2 when they launch nothing), so each case proves which kernel ran.
"""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from test_gemm_bounds_gpu import _SENTINEL, bound_check

U = 2.0 ** -24
GN_FAMILIES = ("flat", "offset", "channel-spread", "frames", "tiny-var", "silu-tail")
_WORST = {}                    # path -> (worst bound ratio, case), printed at the end of the module


# ---------------------------------------------------------------------------------------------------------- references
def _silu64(y):
    return y / (1 + torch.exp(-y))


def _act_terms(y, D, tanh_form=False):
    """(s'(y), e_act(y)) of a SiLU: y / (1 + __expf(-y)) (skinny linear), or 0.5 y (1 + tanh.approx(y / 2)) (GroupNorm)
    when ``tanh_form`` (module docstring)."""
    sig = torch.sigmoid(y)
    ds = (sig * (1 + y * (1 - sig))).abs()
    s1 = torch.clamp(ds + 0.5 * D, max=1.1)
    if tanh_form:
        return s1, 2.0 ** -11.9 * (y * torch.tanh(0.5 * y)).abs() + 2.0 ** -22 * _silu64(y).abs()
    e = (5 + 1.2 * y.abs()) * 2.0 ** -23 * _silu64(y).abs() + 2.0 ** -126
    return s1, torch.where(y < -80, _silu64(y).abs() + 2.0 ** -126, e)


def groupnorm_ref64(x1, x2, NB, HW, G, gamma, beta, eps, silu, n_add, frames=None):
    """(ref, bound without the output rounding) [len(frames) * HW, C1 + C2] of per-frame GroupNorm (+SiLU) of [x1 | x2]
    (exact bf16 values), for the frames listed (default: all)."""
    frames = range(NB) if frames is None else frames
    C = x1.shape[1] + (0 if x2 is None else x2.shape[1])
    cpg = C // G
    refs, bnds = [], []
    gam = gamma.double().view(1, G, cpg)
    bet = beta.double().view(1, G, cpg)
    eps = float(torch.tensor(eps, dtype=torch.float32))
    for n in frames:
        r = slice(n * HW, (n + 1) * HW)
        x = x1[r].double() if x2 is None else torch.cat([x1[r].double(), x2[r].double()], 1)
        x = x.view(HW, G, cpg)
        mu = x.mean((0, 2), keepdim=True)
        d = x - mu
        var = (d * d).mean((0, 2), keepdim=True)
        rstd = (var + eps).rsqrt()
        dmax = d.abs().amax((0, 2), keepdim=True)
        k2 = torch.where(var > 0, dmax * dmax / torch.where(var > 0, var, torch.ones_like(var)), torch.zeros_like(var))
        d_var = (3 * n_add + 8) * U * (1 + k2)
        d_rstd = 0.5 * (d_var * var / (var + eps) + 2 * U) + 4 * U
        d_mean = (2 * n_add + 4) * U * dmax + U * mu.abs()
        z = d * rstd
        y = z * gam + bet
        D = (gam.abs() * (z.abs() * d_rstd + rstd * d_mean)
             + 2.0 ** -23 * ((x.abs() + 2 * mu.abs()) * rstd * gam.abs() + bet.abs() + y.abs()))
        if silu:
            s1, e = _act_terms(y, D, tanh_form=True)
            refs.append(_silu64(y).reshape(HW, C))
            bnds.append((s1 * D + e).reshape(HW, C))
        else:
            refs.append(y.reshape(HW, C))
            bnds.append(D.reshape(HW, C))
    return torch.cat(refs), torch.cat(bnds)


def _gn_block_R(C, target):
    V = C // 8
    r = max(1, target // V)
    while V * r > 1024:
        r -= 1
    return r


def _gn_adds(HW, C, G, S=1):
    """fp32 adds on the longest path of a group's statistics in any of the three kernels (stats / one-launch: R = 256 / V
    pixel lanes, S chunks; cluster: R = 640 / V lanes, at most 8 partials; S = 1 covers a single chunk)."""
    cpg = C // G
    r_min, r_max = _gn_block_R(C, 256), _gn_block_R(C, 640)
    return math.ceil(math.ceil(HW / S) / r_min) + r_max * cpg + max(S, 8) + 8


def layernorm_ref64(x, gamma, beta, eps, pe=None, rpf=0):
    """(ref, bound without the output rounding) of LayerNorm over the rows of x (+ pe[(row // rpf) % len(pe)])."""
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    d = xd - mu
    rstd = ((d * d).mean(1, keepdim=True) + float(torch.tensor(eps, dtype=torch.float32))).rsqrt()
    zg = d * rstd * gamma.double()
    ref = zg + beta.double()
    pa = 0
    if pe is not None:
        p = pe.double()[(torch.arange(x.shape[0], device=x.device) // rpf) % pe.shape[0]]
        ref = ref + p
        pa = p.abs()
    bnd = (2.0 ** -17 * rstd * gamma.double().abs() * xd.abs().amax(1, keepdim=True) + 2.0 ** -18 * zg.abs()
           + 2.0 ** -21 * (beta.double().abs() + pa))
    return ref, bnd


def row_stats_ref64(x, eps):
    """(ref, bound) [rows, 2] = (mean, rstd) of every row, fp32 outputs."""
    xd = x.double()
    mu = xd.mean(1)
    rstd = (((xd - mu[:, None]) ** 2).mean(1) + float(torch.tensor(eps, dtype=torch.float32))).rsqrt()
    ref = torch.stack([mu, rstd], 1)
    bnd = torch.stack([2.0 ** -17 * xd.abs().amax(1), 2.0 ** -18 * rstd + 2.0 ** -17 * xd.abs().amax(1) * rstd ** 2], 1)
    return ref, bnd


def geglu_ref64(x):
    """(ref, bound without the output rounding) of h gelu_erf(g) for x = [h | g]."""
    inner = x.shape[1] // 2
    h, g = x[:, :inner].double(), x[:, inner:].double()
    ref = h * 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))
    return ref, 0.5 * (h * g).abs() * (2.0 ** -22 + 2.0 ** -23 * g.abs()) + 2.0 ** -22 * ref.abs()


def softmax_ref64(x):
    """(ref, bound without the output rounding) of the row softmax of fp32 scores x."""
    xd = x.double()
    t = xd - xd.amax(1, keepdim=True)
    p = torch.softmax(xd, 1)
    e = (2 + 1.2 * t.abs()) * 2.0 ** -23
    E = (p * e).sum(1, keepdim=True)
    n = x.shape[1]
    return p, p * (e + U * t.abs() + E + (n / 256 + 16) * U + 2 * U) + 2.0 ** -126


def timestep_ref(t, dim):
    """The reference's Timesteps(dim, flip_sin_to_cos=True, shift 0) in torch at fp32, before its cast to bf16 -> (ref,
    bound without the cast's rounding)."""
    half = dim // 2
    freq = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    a = t.float()[:, None] * freq[None]
    ref = torch.cat([torch.cos(a), torch.sin(a)], 1).double()
    ad = a.double().abs().repeat(1, 2)
    return ref, 2.0 ** -19 * ad + 2.0 ** -21


def skinny_ref64(x, w, bias, act_in, act_out):
    """(ref, bound) of act_out(act_in(x) W^T + b), fp32 x, bf16 w, fp32 out."""
    xd = x.double()
    a = _silu64(xd) if act_in else xd
    wd = w.double()
    v = a @ wd.t() + (0 if bias is None else bias.double())
    K = x.shape[1]
    D = (K / 32 + 8) * U * (a.abs() @ wd.abs().t()) + (0 if bias is None else U * bias.double().abs())
    if act_in:
        D = D + ((3 + 1.2 * xd.abs()) * 2.0 ** -23 * a.abs()) @ wd.abs().t()
    if not act_out:
        return v, D
    s1, e = _act_terms(v, D)
    return _silu64(v), s1 * D + e


# ------------------------------------------------------------------------------------------------------- data families
def _bf16_exact_around(mu, k, dev):
    """bf16(mu) + k ulp(bf16(mu)) as exact bf16 values."""
    m = mu.bfloat16().float()
    ulp = torch.exp2(torch.floor(torch.log2(m.abs())) - 7)
    return (m + k * ulp).bfloat16()


def gn_inputs(fam, g, NB, HW, C1, C2, G=32, eps=1e-5):
    """bf16 x1 [NB HW, C1], x2 [NB HW, C2] (or None), fp32 gamma / beta [C] on g's device."""
    dev = g.device
    C = C1 + C2
    cpg = C // G
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    ru = lambda *s: torch.rand(*s, device=dev, generator=g)
    gamma, beta = 1 + 0.5 * rn(C), 0.5 * rn(C)
    grp = torch.arange(C, device=dev) // cpg
    if fam == "offset":
        # per (frame, group): mu with random mantissa over 2^-2 .. 2^10 and k uniform in [-K, K], K in {12, 3, 1}
        mu = torch.exp2(torch.randint(-2, 11, (NB, 1, G), device=dev, generator=g).float()) * (1 + ru(NB, 1, G))
        K = torch.tensor([12.0, 3.0, 1.0], device=dev)[torch.randint(0, 3, (NB, 1, G), device=dev, generator=g)]
        k = torch.round((2 * ru(NB, HW, G, cpg) - 1) * K[..., None])
        x = _bf16_exact_around(mu[..., None].expand(NB, HW, G, cpg), k, dev).float()
        near = torch.where(ru(NB, HW, cpg) < 0.01, torch.sign(rn(NB, HW, cpg)) * 4.0, torch.zeros(NB, HW, cpg, device=dev))
        x[:, :, 0] = 1000.0 + near
        x[:, :, 1] = 3.0
        if G > 2:
            x[:, :, 2] = (1000.0 + 4 * rn(NB, HW, cpg)).bfloat16().float()
        x = x.reshape(NB * HW, C)
    elif fam == "channel-spread":
        x = rn(NB * HW, C) * torch.exp2(6.0 * torch.sign(rn(C)))
    elif fam == "frames":
        n = (torch.arange(NB * HW, device=dev) // HW) % 3
        x = (rn(NB * HW, C) + (grp % 4).float()) * (4.0 ** n.float())[:, None] + 3.0 * n.float()[:, None]
    elif fam == "tiny-var":
        k = 0.3 + 2.7 * ru(G)
        x = rn(NB * HW, C) * (math.sqrt(eps) * k)[grp]
    elif fam == "silu-tail":
        x = rn(NB * HW, C)
        gamma, beta = 2 + 3 * ru(C), -12 + 8 * ru(C)
    else:
        x = rn(NB * HW, C)
    x = x.bfloat16()
    return x[:, :C1], (x[:, C1:] if C2 else None), gamma, beta


def ln_inputs(g, rows, C, pe_frames=0):
    dev = g.device
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    x = (rn(rows, C) * torch.exp2(2 * rn(rows, 1)) + 2 * rn(rows, 1)).bfloat16()
    pe = rn(pe_frames, C) if pe_frames else None
    return x, 1 + 0.5 * rn(C), 0.5 * rn(C), pe


# ------------------------------------------------------------------------------------------- CPU model of the kernels
GN_FAULTS = ("frame_shift", "channel_missing", "seam_group_shift", "eps_swap", "sample_var", "no_shift",
             "silu_exp_form", "silu_unhalved")
LN_FAULTS = ("pe_next_frame", "ln_mean_short")
GEGLU_FAULTS = ("gelu_tanh",)
FAULTS = GN_FAULTS + LN_FAULTS + GEGLU_FAULTS
_NOT_FAULTS = ("silu_exp_form",)   # variants a correct kernel may use: they must pass


def _chan(c1, m1, q1, c2, m2, q2):
    """Chan et al. merge of (count, mean, M2) partials in fp32, the kernel's formula; empty partials (c2 == 0) skip."""
    tot = c1 + c2
    delta = m2 - m1
    ok = c2 > 0
    safe = torch.where(ok, tot, torch.ones_like(tot))
    m = torch.where(ok, m1 + delta * (c2 / safe), m1)
    q = torch.where(ok, q1 + q2 + delta * delta * (c1 * c2 / safe), q1)
    return torch.where(ok, tot, c1), m, q


def emulate_groupnorm(x1, x2, NB, HW, G, gamma, beta, eps, silu, S, fault=None):
    """The kernels' arithmetic in torch: statistics of x - pivot (pivot = pixel 0 of the group's first channel) in fp32 per
    pixel chunk, the S partials merged by Chan's formula in the order of gn_apply_body (lane s holds partials s, s + 32,
    ..., then a shuffle-down tree), fp32 apply, SiLU 0.5 y (1 + tanh(y / 2)) with tanh rounded to 11 significant bits (a
    relative error of up to 2^-12, the size of tanh.approx's), bf16 output.  ``fault`` injects one bug:
      frame_shift      : frame n normalised with the statistics of frame n + 1;
      channel_missing  : the last channel of every group left out of its statistics;
      seam_group_shift : channels of x2 normalised with the statistics of the next group;
      eps_swap         : eps 1e-5 where 1e-6 is asked for;
      sample_var       : M2 / (N - 1);
      no_shift         : sums of x and x^2 (no pivot);
      silu_exp_form    : (not a fault) y / (1 + e^-y), the exact form: the bound must pass it too;
      silu_unhalved    : sigmoid as 0.5 + 0.5 tanh(y)."""
    x = (x1.float() if x2 is None else torch.cat([x1.float(), x2.float()], 1)).view(NB, HW, -1)
    C = x.shape[2]
    C1 = x1.shape[1]
    cpg = C // G
    xg = x.view(NB, HW, G, cpg)
    piv = torch.zeros(NB, 1, G, 1) if fault == "no_shift" else xg[:, :1, :, :1]
    d = xg - piv
    use = cpg - 1 if fault == "channel_missing" else cpg
    d = d[..., :use]
    chunk = (HW + S - 1) // S
    lanes = [[] for _ in range(32)]
    for s in range(S):
        p0, p1 = s * chunk, min(HW, (s + 1) * chunk)
        if p1 <= p0:
            part = (torch.zeros(NB, G), torch.zeros(NB, G), torch.zeros(NB, G))
        else:
            ds = d[:, p0:p1]
            a = ds.sum((1, 3), dtype=torch.float32)
            b = (ds * ds).sum((1, 3), dtype=torch.float32)
            cnt = torch.full((NB, G), float((p1 - p0) * use))
            mean = a / cnt
            part = (cnt, mean, torch.clamp(b - a * mean, min=0))
        lanes[s % 32].append(part)
    st = []
    for L in lanes:
        acc = (torch.zeros(NB, G), torch.zeros(NB, G), torch.zeros(NB, G))
        for p in L:
            acc = _chan(*acc, *p)
        st.append(acc)
    for off in (16, 8, 4, 2, 1):
        st = [_chan(*st[i], *st[i + off]) if i + off < 32 else st[i] for i in range(32)]
    cnt, mean, m2 = st[0]
    mean = mean + piv.view(NB, G)
    if fault == "sample_var":
        cnt = cnt - 1
    e = 1e-5 if fault == "eps_swap" and eps == 1e-6 else eps
    rstd = torch.rsqrt(m2 / cnt + e)
    if fault == "frame_shift":
        mean, rstd = mean.roll(-1, 0), rstd.roll(-1, 0)
    gidx = torch.arange(C) // cpg
    if fault == "seam_group_shift":
        gidx = torch.where(torch.arange(C) >= C1, torch.clamp(gidx + 1, max=G - 1), gidx)
    sc = rstd[:, gidx] * gamma.float()
    sh = beta.float() - mean[:, gidx] * sc
    y = x * sc[:, None] + sh[:, None]
    if silu:
        if fault == "silu_exp_form":
            y = y / (1 + torch.exp(-y))
        else:
            m, e = torch.frexp(torch.tanh(y if fault == "silu_unhalved" else 0.5 * y))
            y = y * (0.5 + 0.5 * torch.ldexp(torch.round(m * 2.0 ** 11) / 2.0 ** 11, e))
    return y.reshape(NB * HW, C).bfloat16()


def emulate_layernorm(x, gamma, beta, eps, pe=None, rpf=0, fault=None):
    """fp32 two-pass LayerNorm (+ pe) -> bf16.  pe_next_frame: PE row of frame f + 1; ln_mean_short: the mean over C - 8
    channels."""
    xf = x.float()
    C = x.shape[1]
    mean = (xf[:, :C - 8] if fault == "ln_mean_short" else xf).sum(1, keepdim=True) / C
    q = ((xf - mean) ** 2).sum(1, keepdim=True)
    y = (xf - mean) * torch.rsqrt(q / C + eps) * gamma + beta
    if pe is not None:
        f = torch.arange(x.shape[0]) // rpf + (1 if fault == "pe_next_frame" else 0)
        y = y + pe[f % pe.shape[0]]
    return y.bfloat16()


def emulate_geglu(x, fault=None):
    inner = x.shape[1] // 2
    h, g = x[:, :inner].float(), x[:, inner:].float()
    return (h * F.gelu(g, approximate="tanh" if fault == "gelu_tanh" else "none")).bfloat16()


# (family, kind, shape): gn kinds "seam" (C1 640 | C2 320, 32 groups of 30: the seam inside group 21, 3 frames, 2 chunks)
# and "small" (HW 16, C 48 | 16, cpg 2: one 16-byte vector spans 4 groups, N = 32 per group)
_GN_CPU = {"seam": (3, 64, 640, 320, 2), "small": (3, 16, 48, 16, 1)}


def _cpu_cases():
    cases = [(f, "gn", k) for f in GN_FAMILIES for k in _GN_CPU]
    return cases + [("pe", "ln", None), ("gate", "geglu", None)]


def _cpu_case(fam, kind, shape, g):
    """-> (run(fault) -> out, ref, bnd)."""
    if kind == "gn":
        NB, HW, C1, C2, S = _GN_CPU[shape]
        eps = 1e-6 if fam in ("tiny-var", "flat") else 1e-5
        silu = fam in ("silu-tail", "offset", "frames")
        x1, x2, gam, bet = gn_inputs(fam, g, NB, HW, C1, C2, eps=eps)
        ref, bnd = groupnorm_ref64(x1, x2, NB, HW, 32, gam, bet, eps, silu, _gn_adds(HW, C1 + C2, 32, S))
        return (lambda fault: emulate_groupnorm(x1, x2, NB, HW, 32, gam, bet, eps, silu, S, fault)), ref, bnd
    if kind == "ln":
        rows, C, pf, rpf = 7 * 13, 320, 4, 13
        x, gam, bet, pe = ln_inputs(g, rows, C, pf)
        ref, bnd = layernorm_ref64(x, gam, bet, 1e-5, pe, rpf)
        return (lambda fault: emulate_layernorm(x, gam, bet, 1e-5, pe, rpf, fault)), ref, bnd
    x = (torch.randn(200, 2 * 256, generator=g) * torch.cat([torch.ones(256), 3 * torch.ones(256)])).bfloat16()
    ref, bnd = geglu_ref64(x)
    return (lambda fault: emulate_geglu(x, fault)), ref, bnd


def _applies(fault, kind):
    return fault in {"gn": GN_FAULTS, "ln": LN_FAULTS, "geglu": GEGLU_FAULTS}[kind]


def test_norm_bound_rejects_injected_faults():
    """The faithful model stays within the bound on every family, every injected fault fails the bound or the global
    criterion on at least one family, and every family catches at least one fault."""
    caught = {f: [] for f in FAULTS if f not in _NOT_FAULTS}
    cases = _cpu_cases()
    for i, (fam, kind, shape) in enumerate(cases):
        run, ref, bnd = _cpu_case(fam, kind, shape, torch.Generator().manual_seed(200 + i))
        worst, rel, where = bound_check(run(None), ref, bnd)
        print(f"faithful model {kind:5s} {fam:14s} {shape or '':5s}: worst ratio {worst:.3f}, rel {rel:.2e}")
        assert worst <= 1 and rel < 5e-3, (fam, kind, shape, where, rel)
        for fault in FAULTS:
            if not _applies(fault, kind):
                continue
            worst, rel, where = bound_check(run(fault), ref, bnd)
            if fault in _NOT_FAULTS:
                assert worst <= 1 and rel < 5e-3, (fault, fam, kind, shape, where, rel)
                continue
            if worst > 1 or not rel < 5e-3:
                caught[fault].append((fam, f"{kind} {shape}" if shape else kind, worst, rel, where))
    for fault, hits in caught.items():
        print(f"{fault:17s} rejected on " + ", ".join(f"{f} ({k}: ratio {w:.3g}, rel {r:.2e})" for f, k, w, r, _ in hits))
        assert hits, f"{fault} passes every family"
    for fam, kind, shape in cases:
        assert any(h[0] == fam for hits in caught.values() for h in hits), f"{kind} / {fam} catches no fault"


def test_cpu_references_agree():
    """The fp64 references against torch's own GroupNorm / LayerNorm / softmax / GELU in fp64."""
    g = torch.Generator().manual_seed(3)
    NB, HW, C1, C2 = 3, 20, 40, 24
    x1, x2, gam, bet = gn_inputs("frames", g, NB, HW, C1, C2)
    x = torch.cat([x1, x2], 1).double()
    for silu in (False, True):
        ref, _ = groupnorm_ref64(x1, x2, NB, HW, 32, gam, bet, 1e-5, silu, 1)
        t = F.group_norm(x.view(NB, HW, -1).transpose(1, 2), 32, gam.double(), bet.double(), 1e-5)
        t = t.transpose(1, 2).reshape(NB * HW, -1)
        torch.testing.assert_close(ref, F.silu(t) if silu else t)
    xl, gl, bl, pe = ln_inputs(g, 30, 64, 3)
    ref, _ = layernorm_ref64(xl, gl, bl, 1e-5, pe, 7)
    want = F.layer_norm(xl.double(), (64,), gl.double(), bl.double(), 1e-5) + pe.double()[(torch.arange(30) // 7) % 3]
    torch.testing.assert_close(ref, want)
    xs = torch.randn(5, 12, generator=g) * 30
    torch.testing.assert_close(softmax_ref64(xs)[0], torch.softmax(xs.double(), 1))
    xg = torch.randn(6, 16, generator=g).bfloat16()
    torch.testing.assert_close(geglu_ref64(xg)[0], xg[:, :8].double() * F.gelu(xg[:, 8:].double()))


# ---------------------------------------------------------------------------------------- validation without a device
_VALIDATION = r"""
import ctypes, sys
sys.path.insert(0, sys.argv[1])
from vexpress_b200 import _ffi
L = _ffi.lib()
buf = ctypes.create_string_buffer(1 << 16)
a = (ctypes.addressof(buf) + 255) // 256 * 256
P = lambda off=0: ctypes.c_void_p(a + off)
ll, i, f = ctypes.c_longlong, ctypes.c_int, ctypes.c_float
ok = []
def expect(name, rc, what):
    msg = L.vx_last_error().decode()
    print(name, rc, msg)
    assert rc == 1 and what in msg, (name, rc, msg)
    ok.append(name)
# (misaligned pointer, misaligned leading dimension) per entry point; x1 / x2 / out / gamma / beta are separate blocks
for off, ld in ((2, 64), (0, 68)):
    expect("vx_layernorm", L.vx_layernorm(P(off), ll(ld), ll(4), i(64), P(8192), P(8448), f(1e-5), None, i(0), i(0),
                                          P(16384), ll(64), None), "16-byte aligned")
    expect("vx_layernorm_fp8", L.vx_layernorm_fp8(P(off), ll(ld), ll(4), i(64), P(8192), P(8448), f(1e-5), None, i(0), i(0),
                                                  P(16384), ll(64), P(24576), None), "16-byte aligned")
    expect("vx_row_stats", L.vx_row_stats(P(off), ll(ld), ll(4), i(64), f(1e-5), P(16384), None), "16-byte aligned")
    expect("vx_geglu", L.vx_geglu(P(off), ll(ld + 64), ll(4), i(64), P(16384), ll(64), None), "16-byte aligned")
    gn = (P(off), ll(ld), i(64), P(4096), ll(64), i(32))
    expect("vx_groupnorm_stats", L.vx_groupnorm_stats(*gn, i(2), i(16), i(32), i(1), P(16384), None), "16-byte aligned")
    expect("vx_groupnorm_apply", L.vx_groupnorm_apply(*gn, i(2), i(16), i(32), i(1), P(16384), P(8192), P(8448), f(1e-5),
                                                      i(1), P(20480), ll(96), None), "16-byte aligned")
    expect("vx_groupnorm_fused", L.vx_groupnorm_fused(*gn, i(2), i(16), i(32), i(1), P(16384), P(12288), P(8192), P(8448),
                                                      f(1e-5), i(1), P(20480), ll(96), None), "16-byte aligned")
    expect("vx_groupnorm_cluster", L.vx_groupnorm_cluster(*gn, i(2), i(16), i(32), P(8192), P(8448), f(1e-5), i(1),
                                                          P(20480), ll(96), None), "16-byte aligned")
    # the second source, and the output, each on their own
    gn2 = (P(0), ll(64), i(64), P(4096 + off), ll(ld), i(32))
    expect("vx_groupnorm_stats x2", L.vx_groupnorm_stats(*gn2, i(2), i(16), i(32), i(1), P(16384), None), "16-byte aligned")
    expect("vx_groupnorm_cluster out", L.vx_groupnorm_cluster(P(0), ll(64), i(64), P(4096), ll(64), i(32), i(2), i(16), i(32),
                                                              P(8192), P(8448), f(1e-5), i(1), P(20480 + off), ll(ld + 32),
                                                              None), "16-byte aligned")
# wider than the kernels' register file allows
wide = (P(0), ll(8192), i(8192), None, ll(0), i(0), i(2), i(64), i(32))
expect("vx_groupnorm_stats wide", L.vx_groupnorm_stats(*wide, i(1), P(16384), None), "too wide")
expect("vx_groupnorm_apply wide", L.vx_groupnorm_apply(*wide, i(1), P(16384), P(8192), P(8448), f(1e-5), i(1), P(20480),
                                                       ll(8192), None), "too wide")
expect("vx_groupnorm_fused wide", L.vx_groupnorm_fused(*wide, i(1), P(16384), P(12288), P(8192), P(8448), f(1e-5), i(1),
                                                       P(20480), ll(8192), None), "too wide")
expect("vx_groupnorm_cluster wide", L.vx_groupnorm_cluster(*wide, P(8192), P(8448), f(1e-5), i(1), P(20480), ll(8192),
                                                           None), "too wide")
for off, ld in ((4, 64), (0, 66)):
    expect("vx_softmax_rows", L.vx_softmax_rows(P(off), ll(ld), ll(4), i(64), P(16384), ll(64), None), "16-byte aligned")
print("rejected", len(ok))
"""


def test_misaligned_operands_rejected_without_device(tmp_path):
    """Every norm / activation entry point rejects a misaligned pointer or leading dimension, and the GroupNorm entries a
    C wider than their kernels can run, with its error code and message before any CUDA call: run with no device
    visible, a missing check could only end in a launch error."""
    lib = os.path.join(os.path.dirname(__file__), "..", "v-express_b200", "lib", "libvxb200.so")
    if not os.path.exists(lib):
        pytest.skip("libvxb200.so not built")
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _VALIDATION, root], env=env, capture_output=True, text=True, timeout=120)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0 and "rejected 26" in r.stdout


def test_ops_wrappers_reject_misaligned_views():
    """ops raises ValueError on the layouts the entry points reject, before it reaches the library."""
    from vexpress_b200 import ops
    x = torch.zeros(16, 72, dtype=torch.bfloat16)
    g32 = torch.ones(64)
    with pytest.raises(ValueError):
        ops.groupnorm(x[:, 4:68], 1, 16, g32, g32, 1e-5, True)                  # 8-byte offset
    with pytest.raises(ValueError):
        ops.groupnorm(x[:, :32], 1, 16, g32, g32, 1e-5, True, x2=x[:, 36:68])  # x2 8-byte offset
    with pytest.raises(ValueError):
        ops.layernorm(x[:, 4:68], g32, g32)
    with pytest.raises(ValueError):
        ops.layernorm_fp8(x[:, 4:68], g32, g32)
    with pytest.raises(ValueError):
        ops.row_stats(x[:, 4:68])
    with pytest.raises(ValueError):
        ops.geglu(x[:, 4:68])
    with pytest.raises(ValueError):
        ops.softmax_rows(torch.zeros(4, 70)[:, 2:66])
    y = torch.zeros(16, 68, dtype=torch.bfloat16)                                 # row stride 68: not a multiple of 8
    with pytest.raises(ValueError):
        ops.layernorm(y[:, :64], g32, g32)
    with pytest.raises(ValueError):
        ops.groupnorm(y[:, :64], 1, 16, g32, g32, 1e-5, True)


# ------------------------------------------------------------------------------------------------------------ GPU cases
# (NB, HW, C1, C2, eps, silu) of every GroupNorm the UNet and ReferenceNet issue at configs[0] (512 x 512, 2 x 4 frames)
# and at 768 x 768 (2 x 16 frames), recorded with the shape-checking fake ops of tests/test_host_cpu.py; the VAE decoder's
# (mid block and up blocks of 512 / 512 / 256 / 128 channels, eps 1e-6) follow its structure at one frame per launch.  The
# decoder runs 16 frames per launch (the pipeline's vae_chunk), which changes the dispatch's S: those shapes, and the tail
# chunks of 1..15 frames, are checked frame by frame in tests/test_vae_chunk_bounds_gpu.py.
GN_UNET = [
    (1, 64, 1280, 0, 1e-05, True), (1, 64, 1280, 1280, 1e-05, True), (1, 256, 640, 0, 1e-05, True),
    (1, 256, 1280, 0, 1e-05, True), (1, 256, 1280, 640, 1e-05, True), (1, 256, 1280, 1280, 1e-05, True),
    (1, 1024, 320, 0, 1e-05, True), (1, 1024, 640, 0, 1e-05, True), (1, 1024, 640, 320, 1e-05, True),
    (1, 1024, 640, 640, 1e-05, True), (1, 1024, 1280, 640, 1e-05, True), (1, 4096, 320, 0, 1e-05, True),
    (1, 4096, 320, 320, 1e-05, True), (1, 4096, 640, 320, 1e-05, True), (8, 64, 1280, 0, 1e-06, False),
    (8, 64, 1280, 0, 1e-05, True), (8, 64, 1280, 1280, 1e-05, True), (8, 256, 640, 0, 1e-05, True),
    (8, 256, 1280, 0, 1e-06, False), (8, 256, 1280, 0, 1e-05, True), (8, 256, 1280, 640, 1e-05, True),
    (8, 256, 1280, 1280, 1e-05, True), (8, 1024, 320, 0, 1e-05, True), (8, 1024, 640, 0, 1e-06, False),
    (8, 1024, 640, 0, 1e-05, True), (8, 1024, 640, 320, 1e-05, True), (8, 1024, 640, 640, 1e-05, True),
    (8, 1024, 1280, 640, 1e-05, True), (8, 4096, 320, 0, 1e-06, False), (8, 4096, 320, 0, 1e-05, True),
    (8, 4096, 320, 320, 1e-05, True), (8, 4096, 640, 320, 1e-05, True),
    (1, 64, 1280, 0, 1e-06, False), (1, 256, 1280, 0, 1e-06, False), (1, 1024, 640, 0, 1e-06, False),
    (1, 4096, 320, 0, 1e-06, False)]
GN_UNET_768 = [
    (1, 144, 1280, 0, 1e-05, True), (1, 144, 1280, 1280, 1e-05, True), (1, 576, 640, 0, 1e-05, True),
    (1, 576, 1280, 0, 1e-05, True), (1, 576, 1280, 640, 1e-05, True), (1, 576, 1280, 1280, 1e-05, True),
    (1, 2304, 320, 0, 1e-05, True), (1, 2304, 640, 0, 1e-05, True), (1, 2304, 640, 320, 1e-05, True),
    (1, 2304, 640, 640, 1e-05, True), (1, 2304, 1280, 640, 1e-05, True), (1, 9216, 320, 0, 1e-05, True),
    (1, 9216, 320, 320, 1e-05, True), (1, 9216, 640, 320, 1e-05, True), (32, 144, 1280, 0, 1e-06, False),
    (32, 144, 1280, 0, 1e-05, True), (32, 144, 1280, 1280, 1e-05, True), (32, 576, 640, 0, 1e-05, True),
    (32, 576, 1280, 0, 1e-06, False), (32, 576, 1280, 0, 1e-05, True), (32, 576, 1280, 640, 1e-05, True),
    (32, 576, 1280, 1280, 1e-05, True), (32, 2304, 320, 0, 1e-05, True), (32, 2304, 640, 0, 1e-06, False),
    (32, 2304, 640, 0, 1e-05, True), (32, 2304, 640, 320, 1e-05, True), (32, 2304, 640, 640, 1e-05, True),
    (32, 2304, 1280, 640, 1e-05, True), (32, 9216, 320, 0, 1e-06, False), (32, 9216, 320, 0, 1e-05, True),
    (32, 9216, 320, 320, 1e-05, True), (32, 9216, 640, 320, 1e-05, True),
    (1, 144, 1280, 0, 1e-06, False), (1, 576, 1280, 0, 1e-06, False), (1, 2304, 640, 0, 1e-06, False),
    (1, 9216, 320, 0, 1e-06, False)]
GN_VAE = [(1, s * s * m, C, 0, 1e-06, silu) for s in (64, 96)
          for m, C, silu in ((1, 512, True), (1, 512, False), (4, 512, True), (16, 512, True), (16, 256, True),
                             (64, 256, True), (64, 128, True))]
GN_PRODUCTION = sorted(set(GN_UNET + GN_UNET_768 + GN_VAE))
# LayerNorm (rows, C, pe frames, rows per frame), same calls
LN_PRODUCTION = [(512, 1280, 0, 0), (512, 1280, 4, 64), (2048, 1280, 0, 0), (2048, 1280, 4, 256), (8192, 640, 0, 0),
                 (8192, 640, 4, 1024), (32768, 320, 0, 0), (32768, 320, 4, 4096), (64, 1280, 0, 0), (256, 1280, 0, 0),
                 (1024, 640, 0, 0), (4096, 320, 0, 0), (4608, 1280, 16, 144), (18432, 1280, 16, 576),
                 (73728, 640, 16, 2304), (294912, 320, 0, 0), (294912, 320, 16, 9216), (144, 1280, 0, 0),
                 (9216, 320, 0, 0)]
# edges: HW < 32 (one chunk) with cpg 2 (one 16-byte vector spans 4 groups), HW that no cluster size divides, the x1 | x2
# seam inside a group (cpg 30), the widest C the kernels take (4096: C / 8 = 512 threads, cpg 128), HW of several uneven
# chunks, a wide second source
GN_EDGES = [(3, 16, 48, 16), (3, 50, 64, 0), (2, 49, 320, 0), (4, 64, 640, 320), (2, 64, 4096, 0), (3, 1000, 320, 0),
            (2, 4096, 1280, 1280)]


@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture(scope="module", autouse=True)
def _worst_ratio_summary():
    yield
    for path, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {path:18s} {worst:.3f}  ({case})")


def _gpu():
    from test_gemm_bounds_gpu import _bordered, _border_untouched, _in_nan, _INNER
    return _bordered, _border_untouched, _in_nan, _INNER


def _record(path, case, fam, worst, rel, where, out, border):
    print(f"{path:18s} {case} {fam:14s}: worst ratio {worst:.3f}, rel {rel:.2e}")
    if worst > _WORST.get(path, (-1.0, ""))[0]:
        _WORST[path] = (worst, f"{case} {fam}")
    bad = []
    if not worst <= 1:
        bad.append(f"bound exceeded, {where}")
    if not rel < 5e-3:
        bad.append(f"global rel {rel:.3e}")
    if torch.isnan(out.float()).any():
        bad.append("NaN left in the output")
    if border:
        bad.append(border)
    return f"{path} {case} {fam}: " + "; ".join(bad) if bad else ""


def _judge(path, case, fam, out, ref, bnd, border="", bf16_out=True):
    torch.cuda.synchronize()
    worst, rel, where = bound_check(out, ref, bnd, bf16_out)
    return _record(path, case, fam, worst, rel, where, out, border)


def _seed(*ints):
    s = 0
    for i in ints:
        s = (s * 1000003 + int(round(float(i) * 1e6)) % (1 << 40)) % (1 << 31)
    return s


def _cluster_fits(NB, HW, C, G=32):
    """vx_groupnorm_cluster's rule: the frame in <= 8 CTAs' shared memory, one wave of clusters."""
    R = _gn_block_R(C, 640)
    fixed = (2 * R * C + 5 * G + 2 * C) * 4
    for cl in (1, 2, 4, 8):
        if HW % cl:
            return False
        if HW // cl * C * 2 + fixed <= 200 * 1024:
            return NB * cl <= torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return False


def _gn_run(ops, path, x1, x2, NB, HW, gam, bet, eps, silu, out, G=32):
    """One GroupNorm through ``path``: cluster / fused / pair (entry points called directly) or dispatch (ops.groupnorm,
    also under VX_GN_FRAMES) -> (return code, S the statistics were chunked into, workspace to keep alive)."""
    from vexpress_b200 import _ffi
    from vexpress_b200._ffi import c_float, c_int, c_ll, ptr, stream_ptr
    L = _ffi.lib()
    C1 = x1.shape[1]
    C2 = 0 if x2 is None else x2.shape[1]
    C = C1 + C2
    head = (ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), c_ll(0 if x2 is None else x2.stride(0)), c_int(C2),
            c_int(NB), c_int(HW), c_int(G))
    tail = (ptr(gam), ptr(bet), c_float(eps), c_int(int(silu)), ptr(out), c_ll(out.stride(0)), stream_ptr())
    S = ops._gn_S(NB, HW, C)
    ws = torch.empty(NB * S * G * 3, device="cuda", dtype=torch.float32)
    if path == "cluster":
        return L.vx_groupnorm_cluster(*head, *tail), 1, ws
    if path == "fused":
        return L.vx_groupnorm_fused(*head, c_int(S), ptr(ws), ptr(ops._gn_counters(x1.device, NB)), *tail), S, ws
    if path == "pair":
        rc = L.vx_groupnorm_stats(*head, c_int(S), ptr(ws), stream_ptr())
        return rc or L.vx_groupnorm_apply(*head, c_int(S), ptr(ws), *tail), S, ws
    ops.groupnorm(x1, NB, HW, gam, bet, eps, silu, x2=x2, groups=G, out=out)
    grp = int(os.environ.get("VX_GN_FRAMES", "0"))
    if 0 < grp < NB:
        return 0, ops._gn_S(grp, HW, C), ws
    return 0, (1 if ops._GN_CLUSTER and _cluster_fits(NB, HW, C, G) else S), ws


def _run_gn(ops, path, fams, NB, HW, C1, C2, eps=1e-5, silu=True, expect_rc=0):
    """GroupNorm of each family through ``path`` with x1 / x2 interior views of separate NaN-filled buffers and out inside
    a sentinel border; the reference and the judgement go frame block by frame block."""
    _bordered, _border_untouched, _in_nan, _INNER = _gpu()
    C = C1 + C2
    case = f"NB {NB} HW {HW} C {C1}+{C2} eps {eps:g} silu {int(silu)}"
    fails = []
    for fam in fams:
        e = eps
        if fam.startswith("tiny-var"):
            fam, e = "tiny-var", float(fam.split("@")[1]) if "@" in fam else eps
        g = torch.Generator(device="cuda").manual_seed(_seed(NB, HW, C1, C2, GN_FAMILIES.index(fam), e))
        x1, x2, gam, bet = gn_inputs(fam, g, NB, HW, C1, C2, eps=e)
        s = silu or fam == "silu-tail"
        obuf, out = _bordered(NB * HW, C)
        rc, S, ws = _gn_run(ops, path, _in_nan(x1), _in_nan(x2), NB, HW, gam, bet, e, s, out)
        assert rc == expect_rc, f"{path} {case}: return code {rc}, expected {expect_rc}"
        if rc:
            return
        torch.cuda.synchronize()
        n_add = _gn_adds(HW, C, 32, S)
        step = max(1, (1 << 24) // (HW * C))
        worst, where, num, den = 0.0, "", 0.0, 0.0
        for n0 in range(0, NB, step):
            fr = range(n0, min(NB, n0 + step))
            ref, bnd = groupnorm_ref64(x1, x2, NB, HW, 32, gam, bet, e, s, n_add, fr)
            o = out[n0 * HW:fr[-1] * HW + HW]
            w, _, wh = bound_check(o, ref, bnd)
            num += float((o.double() - ref).norm()) ** 2
            den += float(ref.norm()) ** 2
            if w > worst or not where:
                worst, where = w, f"frame block {n0}: {wh}"
        rel = math.sqrt(num / den) if den > 0 else math.sqrt(num)
        fails.append(_record(f"groupnorm {path}", case, f"{fam}@{e:g}" if fam == "tiny-var" else fam, worst, rel, where,
                             out, _border_untouched(obuf, _INNER)))
        del ws
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


GN_ALL = ("flat", "offset", "channel-spread", "frames", "tiny-var@1e-05", "tiny-var@1e-06", "silu-tail")


@pytest.mark.gpu
@pytest.mark.parametrize("NB,HW,C1,C2", GN_EDGES)
@pytest.mark.parametrize("path", ["cluster", "fused", "pair"])
def test_groupnorm_paths_within_bound(ops, path, NB, HW, C1, C2):
    """Every family through each kernel on its own.  The cluster entry must launch (0) exactly where its rule says the
    frame fits, and decline (2) elsewhere."""
    rc = 0 if path != "cluster" or _cluster_fits(NB, HW, C1 + C2) else 2
    _run_gn(ops, path, GN_ALL, NB, HW, C1, C2, silu=True, expect_rc=rc)
    _run_gn(ops, path, ("flat", "offset"), NB, HW, C1, C2, eps=1e-6, silu=False, expect_rc=rc)


@pytest.mark.gpu
@pytest.mark.parametrize("grp", [1, 2, 3])
def test_groupnorm_frames_mode_within_bound(ops, monkeypatch, grp):
    """VX_GN_FRAMES: the statistics / apply pair over groups of frames (a last group shorter than the others at 2, 3)."""
    monkeypatch.setenv("VX_GN_FRAMES", str(grp))
    _run_gn(ops, "frames", ("flat", "offset", "frames", "silu-tail"), 5, 1024, 640, 320)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,HW,C1,C2,eps,silu", GN_PRODUCTION)
def test_groupnorm_production_within_bound(ops, NB, HW, C1, C2, eps, silu):
    """The default dispatch (ops.groupnorm) at every shape the UNet, ReferenceNet and VAE decoder issue."""
    fams = ("flat", "offset", "silu-tail") if silu else ("flat", "offset")
    _run_gn(ops, "dispatch", fams if NB * HW * (C1 + C2) <= (1 << 28) else fams[:2], NB, HW, C1, C2, eps, silu)


# ---- LayerNorm, row statistics
@pytest.fixture
def ln_v1():
    """ln_v1(True / False) sets VX_LN_V1 (every C on the one-warp-per-row kernel) and makes the library re-read it."""
    from vexpress_b200 import _ffi
    before = os.environ.get("VX_LN_V1")

    def switch(on):
        if on:
            os.environ["VX_LN_V1"] = "1"
        else:
            os.environ.pop("VX_LN_V1", None)
        _ffi.lib().vx_norm_reload_env()

    yield switch
    if before is None:
        os.environ.pop("VX_LN_V1", None)
    else:
        os.environ["VX_LN_V1"] = before
    _ffi.lib().vx_norm_reload_env()


def _run_ln(ops, path, rows, C, pe_frames=0, rpf=0):
    _bordered, _border_untouched, _in_nan, _INNER = _gpu()
    g = torch.Generator(device="cuda").manual_seed(_seed(rows, C, pe_frames, rpf))
    x, gam, bet, pe = ln_inputs(g, rows, C, pe_frames)
    obuf, out = _bordered(rows, C)
    ops.layernorm(_in_nan(x), gam, bet, 1e-5, pe=pe, rows_per_frame=rpf, out=out)
    ref, bnd = layernorm_ref64(x, gam, bet, 1e-5, pe, rpf)
    m = _judge(path, f"rows {rows} C {C} pe {pe_frames} x {rpf}", "pe" if pe_frames else "flat", out, ref, bnd,
               _border_untouched(obuf, _INNER))
    assert not m, m


@pytest.mark.gpu
@pytest.mark.parametrize("pe", [False, True])
@pytest.mark.parametrize("v1", [False, True])
@pytest.mark.parametrize("rows", [1, 3, 777, 4096 + 13])
@pytest.mark.parametrize("C", [320, 640, 1280])
def test_layernorm5_widths_within_bound(ops, ln_v1, C, rows, v1, pe):
    """The transformer widths on layernorm5_kernel and (VX_LN_V1) on the generic kernel; row counts that leave a partial
    row set; PE with 13 rows per frame and 4 PE rows for more frames than that."""
    ln_v1(v1)
    _run_ln(ops, "layernorm v1" if v1 else "layernorm5", rows, C, 4 if pe else 0, 13 if pe else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("pe", [False, True])
@pytest.mark.parametrize("C", [8, 64, 256, 264, 768, 1024, 2048])
def test_layernorm_generic_within_bound(ops, C, pe):
    """Every MAXV bucket of the one-warp-per-row kernel and the widths on both sides of its edges."""
    _run_ln(ops, "layernorm generic", 777, C, 4 if pe else 0, 13 if pe else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C,pf,rpf", LN_PRODUCTION)
def test_layernorm_production_within_bound(ops, rows, C, pf, rpf):
    _run_ln(ops, "layernorm", rows, C, pf, rpf)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [8, 64, 320, 640, 1280, 2048])
def test_row_stats_within_bound(ops, C):
    _bordered, _border_untouched, _in_nan, _INNER = _gpu()
    g = torch.Generator(device="cuda").manual_seed(_seed(C, 7))
    x, _, _, _ = ln_inputs(g, 777, C)
    out = ops.row_stats(_in_nan(x))
    ref, bnd = row_stats_ref64(x, 1e-5)
    m = _judge("row_stats", f"rows 777 C {C}", "flat", out, ref, bnd, bf16_out=False)
    assert not m, m


# ---- GEGLU, softmax, time embedding
@pytest.mark.gpu
@pytest.mark.parametrize("rows,inner", [(777, 1280), (100, 5120), (3, 8), (4096, 320)])
def test_geglu_within_bound(ops, rows, inner):
    _bordered, _border_untouched, _in_nan, _INNER = _gpu()
    g = torch.Generator(device="cuda").manual_seed(_seed(rows, inner))
    x = torch.randn(rows, 2 * inner, device="cuda", generator=g)
    x[:, inner:] *= 3
    x = x.bfloat16()
    obuf, out = _bordered(rows, inner)
    ops.geglu(_in_nan(x), out=out)
    ref, bnd = geglu_ref64(x)
    m = _judge("geglu", f"rows {rows} inner {inner}", "gate", out, ref, bnd, _border_untouched(obuf, _INNER))
    assert not m, m


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 1020, 4096, 9216])
def test_softmax_rows_within_bound(ops, n):
    """Row r spreads its scores over 80 r / (rows - 1): from a flat row to scores 80 below the maximum."""
    _bordered, _border_untouched, _in_nan, _INNER = _gpu()
    rows = 33
    g = torch.Generator(device="cuda").manual_seed(_seed(n, 3))
    spread = 80.0 * torch.arange(rows, device="cuda")[:, None] / (rows - 1)
    x = 10 * torch.randn(rows, 1, device="cuda", generator=g) - spread * torch.rand(rows, n, device="cuda", generator=g)
    ld = (n + 24 + 7) // 8 * 8                                   # bf16 rows of whole 16-byte vectors
    obuf = torch.full((rows + 8, ld), _SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    out = obuf[3:3 + rows, 8:8 + n]
    ops.softmax_rows(_in_nan(x), out=out)
    ref, bnd = softmax_ref64(x)
    m = _judge("softmax_rows", f"rows {rows} n {n}", "spread 0-80", out, ref, bnd,
               _border_untouched(obuf, (slice(3, 3 + rows), slice(8, 8 + n))))
    assert not m, m


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [320, 8])
def test_timestep_embed_within_bound(ops, dim):
    t = torch.tensor([999.0, 981.0, 499.0, 20.0, 1.0, 0.0], device="cuda")
    out = ops.timestep_embed(t, dim)
    ref, bnd = timestep_ref(t, dim)
    m = _judge("timestep_embed", f"dim {dim}", "t 0-999", out, ref, bnd)
    assert not m, m


@pytest.mark.gpu
@pytest.mark.parametrize("rows,K,N,act_in,act_out", [(2, 320, 1280, False, True), (2, 1280, 1280, False, False),
                                                     (2, 1280, 3840, True, False), (8, 1280, 640, True, True),
                                                     (1, 8, 16, True, True)])
def test_skinny_linear_within_bound(ops, rows, K, N, act_in, act_out):
    """The time-embedding MLP (linear_1 + SiLU, linear_2) and the SiLU-in projection that feeds every resnet's bias2."""
    g = torch.Generator(device="cuda").manual_seed(_seed(rows, K, N))
    x = 4 * torch.randn(rows, K, device="cuda", generator=g)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    out = ops.skinny_linear(x, w, b, act_in=act_in, act_out=act_out)
    ref, bnd = skinny_ref64(x, w, b, act_in, act_out)
    m = _judge("skinny_linear", f"rows {rows} K {K} N {N} in {int(act_in)} out {int(act_out)}", "N(0, 16)", out, ref, bnd,
               bf16_out=False)
    assert not m, m
