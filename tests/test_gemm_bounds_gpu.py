"""The GEMM / implicit-GEMM convolution kernel (every producer, conv mode and epilogue) and the two small convs around it
(conv_in, conv_out_tc) against an fp64 reference, element by element, under an error bound a correct kernel cannot exceed.

The reference (``linear_ref64``) takes exactly the bf16 / fp32 operands the kernel read and gives, per output element,

    ref      = s (A W^T + b + b2[m // div]) + r
    ref_abs  = |s| (|A| |W|^T + |b| + |b2[m // div]|) + |r|
    prod_abs = |s| |A| |W|^T

with K running over the 9 C (3x3), 9 C at stride 2 or 4 C (upsample folded into four parity-class 2x2 convolutions,
with the packed bf16 weights: that is the operation the kernel performs) im2col columns for convolutions.  The bound is

    |out - ref| <= 2^-8 |ref| + K 2^-22 prod_abs + 2^-20 ref_abs

* 2^-8 |ref|: the one rounding of the output to bf16 (round to nearest, 8 significant bits: unit roundoff 2^-8).  The
  term is reached: a value half an ulp above a power of two rounds by 2^-8 / (1 + 2^-8) of itself, so a correct kernel's
  bf16 outputs reach ratios close to 1 (the CPU model: 0.95 at out 4.094, ref 4.078), and the margin of a bf16 case is
  in the terms below.  Dropped for fp32 output, which makes the check a direct test of the accumulator.
* K 2^-22 prod_abs: the bf16 x bf16 products are exact in fp32; summing K of them in fp32 moves the sum by at most
  K 2^-24 sum |a_k w_k|, times 2 for tensor-core adds that may truncate instead of round, times 2 for the order of the
  partial sums across k-steps and K blocks.
* 2^-20 ref_abs: the few fp32 epilogue operations (+ b, + b2, * s, + r), each a relative 2^-24 of a value no larger
  than ref_abs.
GEGLU (``geglu_ref64``) propagates the accumulation errors dV, dG of the value and gate columns (each
K 2^-22 P + 2^-22 (P + |b|), P = |A| |W|^T of that column) through out = V gelu(G):
|gelu(G)| dV + |V| (d' dG + e_gelu) + dV (1.13 dG + e_gelu), where d' = min(1.13, |gelu'(G)| + 0.8 dG) bounds |gelu'|
on [G - dG, G + dG] (|gelu''| <= 2 phi(0) < 0.8, |gelu'| <= 1.13 everywhere) and e_gelu = |G| (2^-22 + 2^-18 erfc(|G| /
sqrt 2)) + 2^-21 |gelu(G)| covers the kernel's gelu_erf: the A&S 7.1.28 erf (absolute error 3e-7, half of it reaching
gelu as 0.5 |G| 3e-7 < 2^-22 |G|), rcp.approx and the four squarings of (1 + ...)^-16 (a relative 2^-17 of 1 - erf),
and the fp32 products.  The local derivative matters: with the global 1.13 the bound would hide a tanh-GELU, which
differs from the erf form by 10 % around G = -3 where gelu' is tiny.

A correct kernel stays below the bound on any input, so a ratio above 1 is a bug, not a tolerance to widen.  Every case
also keeps the global criterion ||out - ref|| < 5e-3 max(||ref||, ||ref - r||) of tests/test_gemm_gpu.py (the second
norm is the size of the terms the residual cancels in the ``cancel`` family), so that many small errors that add up are
still caught.

The data families are functions of a torch.Generator, shared by the CPU self-test and the GPU cases:
  flat      : N(0, 1) A, W / sqrt(K).
  blocks    : the 64-wide K blocks scaled alternately 2^6 / 2^-6 in A and inversely in W (convs: per channel block, and
              W per tap by 2^(tap % 3 - 1)), so a K block dropped, repeated or paired with the wrong W block moves the
              output by 2^12 of its share.
  cancel    : the residual is -bf16(s (A W^T + b + b2)): the output is a small difference of large terms, which exposes
              rounding before the residual add and residual rows / columns taken from the wrong place.
  frames    : frame n (rows m // div; convs: image n) scaled by 4^(n mod 3), bias2 different in every frame: cross-frame
              tap reads and bias2 rows off by one at a frame boundary inside a tile stand out.
  wide-gate : (GEGLU) gate columns x 4, pre-activations over +-8: the erf tails are used.
``test_bound_rejects_injected_faults`` runs ``emulate_gemm``, a torch model of the kernel's arithmetic with injectable
faults, through the same check: it is the evidence that the GPU cases would catch those faults in the kernel.

Outputs are written into the interior of NaN-filled buffers with a leading dimension larger than N, GEMM operands and
residuals are interior views of NaN-filled buffers (lda / ldw / ldr > K or N, rows past M and N), and conv inputs are the
inner frames of a buffer whose first and last frames are NaN: a read outside the tensor maps turns an output into NaN,
a write outside the output slice shows in the border.
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

FAMILIES = ("flat", "blocks", "cancel", "frames", "wide-gate")
KB = 64                        # K block of the kernel's TMA ring
_SENTINEL = 0x7FC1             # a bf16 NaN no kernel produces: cells around an output slice hold it
_SENTINEL32 = 0x7FC00101       # the fp32 counterpart
_WORST = {}                    # path -> (worst bound ratio, case), printed at the end of the module
_BUDGET = 1 << 29              # bytes of fp64 temporaries per reference chunk


# ---------------------------------------------------------------------------------------------------------- reference
def _f32(x):
    """The fp32 value the kernel receives for a Python float argument."""
    return float(torch.tensor(x, dtype=torch.float32))


def linear_ref64(A, w, bias=None, bias2=None, div=1, scale=1.0, residual=None, row0=0):
    """fp64 (ref, ref_abs, prod_abs) [rows, N] of s (A W^T + b + b2[(row0 + m) // div]) + r for the rows of A [rows, K]
    (any dtype, exact values), w [N, K]."""
    Ad, Wd = A.double(), w.double()
    acc = Ad @ Wd.t()
    pa = Ad.abs() @ Wd.abs().t()
    lin, lin_abs = acc, pa.clone()
    if bias is not None:
        lin = lin + bias.double()
        lin_abs += bias.double().abs()
    if bias2 is not None:
        idx = (row0 + torch.arange(A.shape[0], device=A.device)) // div
        b2 = bias2.reshape(-1, bias2.shape[-1])[idx].double()
        lin = lin + b2
        lin_abs += b2.abs()
    s = _f32(scale)
    ref, ref_abs, prod = s * lin, abs(s) * lin_abs, abs(s) * pa
    if residual is not None:
        ref = ref + residual.double()
        ref_abs += residual.double().abs()
    return ref, ref_abs, prod


def _chunks(rows, K, N):
    step = max(1, _BUDGET // (8 * (K + 4 * N)))
    return [(r0, min(rows, r0 + step)) for r0 in range(0, rows, step)]


def gemm_ref64(a, w, bias=None, a2=None, bias2=None, div=1, scale=1.0, residual=None):
    """linear_ref64 over concat(a, a2), chunked over M -> (ref, ref_abs, prod_abs)."""
    M, N = a.shape[0], w.shape[0]
    out = [torch.empty((M, N), dtype=torch.float64, device=a.device) for _ in range(3)]
    for r0, r1 in _chunks(M, w.shape[1], N):
        A = a[r0:r1] if a2 is None else torch.cat([a[r0:r1], a2[r0:r1]], 1)
        res = None if residual is None else residual[r0:r1]
        for o, t in zip(out, linear_ref64(A, w, bias, bias2, div, scale, res, r0)):
            o[r0:r1] = t
    return tuple(out)


def conv_cols(x, kind="s1", pad_lo=1, par=0, fault=None):
    """im2col of NHWC x [nb, H, W, C] in the kernel's K order -> [nb, Ho, Wo, T C].
    kind s1 : 3x3, stride 1, pad 1, taps (ky, kx) row-major.
    kind s2 : 3x3, stride 2, pad (pad_lo, 1) on both axes (pad_lo 1: nn.Conv2d(padding=1); 0: F.pad(x, (0, 1, 0, 1))).
    kind ups: parity class par = 2 py + px of conv3x3(upsample2x(x)): the 2x2 taps (a, b) read x[i + py - 1 + a, j + px - 1 + b].
    fault (s1 only): conv_frame_leak stacks the frames vertically, so dy taps read the neighbouring frame instead of the
    zero padding; conv_row_wrap lets dx taps wrap to the previous / next pixel row of the same frame."""
    nb, H, W, C = x.shape
    if kind == "s2":
        xp = F.pad(x, (0, 0, pad_lo, 1, pad_lo, 1))
        Ho, Wo = H // 2, W // 2
        return torch.cat([xp[:, ky:ky + 2 * Ho:2, kx:kx + 2 * Wo:2] for ky in range(3) for kx in range(3)], -1)
    if kind == "ups":
        py, px = par >> 1, par & 1
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        return torch.cat([xp[:, py + a:py + a + H, px + b:px + b + W] for a in range(2) for b in range(2)], -1)
    if fault == "conv_frame_leak":
        return conv_cols(x.reshape(1, nb * H, W, C)).reshape(nb, H, W, 9 * C)
    if fault == "conv_row_wrap":
        xh = F.pad(x, (0, 0, 0, 0, 1, 1))
        taps = []
        for ky in range(3):
            flat = F.pad(xh[:, ky:ky + H].reshape(nb, H * W, C), (0, 0, 1, 1))
            taps += [flat[:, kx:kx + H * W].reshape(nb, H, W, C) for kx in range(3)]
        return torch.cat(taps, -1)
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], -1)


def conv_ref64(x, w, bias=None, bias2=None, div=1, scale=1.0, residual=None, kind="s1", pad_lo=1):
    """(ref, ref_abs, prod_abs) [rows, Cout] of the conv in the kernel's output row order (ups: NHWC of the 2x image; the
    parity classes use the packed w [4 Cout, 4 C] blocks).  Frames are im2col'ed one at a time, rows chunked."""
    nb, H, W, C = x.shape
    Cout = w.shape[0] // 4 if kind == "ups" else w.shape[0]
    Ho, Wo = (H // 2, W // 2) if kind == "s2" else (H, W)
    if kind == "ups":
        full = [torch.empty((nb, 2 * H, 2 * W, Cout), dtype=torch.float64, device=x.device) for _ in range(3)]
        for par in range(4):
            for n in range(nb):
                cols = conv_cols(x[n:n + 1], "ups", par=par).reshape(H * W, 4 * C)
                parts = gemm_ref64(cols, w[par * Cout:(par + 1) * Cout], bias)
                for f, t in zip(full, parts):
                    f[n, par >> 1::2, par & 1::2] = t.view(H, W, Cout)
        return tuple(f.reshape(-1, Cout) for f in full)
    hw = Ho * Wo
    out = [torch.empty((nb * hw, Cout), dtype=torch.float64, device=x.device) for _ in range(3)]
    for n in range(nb):
        cols = conv_cols(x[n:n + 1], kind, pad_lo).reshape(hw, -1)
        for r0, r1 in _chunks(hw, cols.shape[1], Cout):
            res = None if residual is None else residual[n * hw + r0:n * hw + r1]
            for o, t in zip(out, linear_ref64(cols[r0:r1], w, bias, bias2, div, scale, res, n * hw + r0)):
                o[n * hw + r0:n * hw + r1] = t
    return tuple(out)


def linear_bound(ref, ref_abs, prod_abs, K):
    """The accumulation and epilogue terms of the bound (everything but the output rounding)."""
    return K * 2.0 ** -22 * prod_abs + 2.0 ** -20 * ref_abs


def _gelu64(G):
    return 0.5 * G * (1 + torch.erf(G / math.sqrt(2)))


def geglu_ref64(a, w, bias):
    """out = (A Wv^T + bv) gelu(A Wg^T + bg) for the UNPACKED w [2 inner, K] (value rows, then gate rows) -> (ref, bound
    without the output rounding), chunked over M."""
    M, K = a.shape
    inner = w.shape[0] // 2
    ref = torch.empty((M, inner), dtype=torch.float64, device=a.device)
    bnd = torch.empty_like(ref)
    for r0, r1 in _chunks(M, K, 4 * w.shape[0]):
        V, _, Pv = linear_ref64(a[r0:r1], w[:inner], bias[:inner])
        G, _, Pg = linear_ref64(a[r0:r1], w[inner:], bias[inner:])
        dV = K * 2.0 ** -22 * Pv + 2.0 ** -22 * (Pv + bias[:inner].double().abs())
        dG = K * 2.0 ** -22 * Pg + 2.0 ** -22 * (Pg + bias[inner:].double().abs())
        ref[r0:r1], bnd[r0:r1] = geglu_propagate(V, G, dV, dG)
    return ref, bnd


def geglu_propagate(V, G, dV, dG):
    """(V gelu(G), bound without the output rounding) for fp64 pre-activations V, G known to within dV, dG."""
    gl = _gelu64(G)
    dgelu = (0.5 * (1 + torch.erf(G / math.sqrt(2))) + G * torch.exp(-0.5 * G * G) / math.sqrt(2 * math.pi)).abs()
    d1 = torch.clamp(dgelu + 0.8 * dG, max=1.13)
    e_gelu = G.abs() * (2.0 ** -22 + 2.0 ** -18 * torch.erfc(G.abs() / math.sqrt(2))) + 2.0 ** -21 * gl.abs()
    return V * gl, (gl.abs() * dV + V.abs() * (d1 * dG + e_gelu) + dV * (1.13 * dG + e_gelu) + 2.0 ** -22 * (V * gl).abs())


def bound_check(out, ref, bnd, bf16_out=True, residual=None):
    """(worst ratio |out - ref| / bound, global relative error, description of the worst element).  NaN counts as an
    infinite ratio; a nonzero error against a zero bound too."""
    o = out.double().reshape(ref.shape).contiguous()
    err = (o - ref).abs()
    bound = bnd + (2.0 ** -8 * ref.abs() if bf16_out else 0)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf).contiguous()
    i = int(ratio.argmax())
    row, col = divmod(i, ref.shape[-1])
    worst = float(ratio.reshape(-1)[i])
    scale = float(ref.norm())
    if residual is not None:
        scale = max(scale, float((ref - residual.double()).norm()))
    rel = float((o - ref).norm()) / scale if scale > 0 else float((o - ref).norm())
    where = (f"worst at (row {row}, column {col}): out {float(o.reshape(-1)[i]):.6g} ref {float(ref.reshape(-1)[i]):.6g} "
             f"bound {float(bound.reshape(-1)[i]):.3g} ratio {worst:.3f}")
    return worst, rel, where


# ------------------------------------------------------------------------------------------------------- data families
def _block_exp(K, blocks_per_tap=None):
    """+6 / -6 per 64-wide K block, alternating (convs: per channel block, the same for every tap)."""
    j = torch.arange(K) // KB
    if blocks_per_tap:
        j = j % blocks_per_tap
    return 6.0 * (1 - 2 * (j % 2)).float()


def gemm_inputs(fam, g, M, K1, K2, N, *, div=1, b2_rows=0, residual=False, geglu=False):
    """bf16 a [M, K1], a2 [M, K2] (or None), w [N, K1 + K2] (GEGLU: unpacked, value rows then gate rows), fp32 bias [N],
    bias2 [b2_rows, N] (or None), bf16 residual [M, N] (or None) on g's device.  ``cancel`` leaves the residual to the
    caller (it needs the reference)."""
    dev = g.device
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    K = K1 + K2
    A, W = rn(M, K), rn(N, K) / math.sqrt(K)
    if fam == "blocks":
        e = _block_exp(K).to(dev)
        A, W = A * torch.exp2(e), W * torch.exp2(-e)
    if fam == "frames":
        A = A * 4.0 ** ((torch.arange(M, device=dev) // div) % 3).float()[:, None]
    if geglu and fam == "wide-gate":
        W[N // 2:] *= 4
    bias = 0.5 * rn(N)
    b2 = None
    if b2_rows:
        b2 = rn(b2_rows, N)
        if fam == "frames":
            b2 = b2 * 4.0 ** (torch.arange(b2_rows, device=dev) % 3).float()[:, None]
    r = rn(M, N).bfloat16() if residual and fam != "cancel" else None
    A = A.bfloat16()
    return A[:, :K1], (A[:, K1:] if K2 else None), W.bfloat16(), bias.bfloat16().float(), b2, r


def conv_inputs(fam, g, NB, H, W, C, Cout, taps=9, b2=False):
    """bf16 x [NB, H, W, C], w [Cout, taps C] (K order (tap, c)), fp32 bias [Cout], bias2 [NB, Cout] (one row per frame,
    or None) on g's device."""
    dev = g.device
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    x, w = rn(NB, H, W, C), rn(Cout, taps, C) / math.sqrt(taps * C)
    if fam == "blocks":
        e = _block_exp(C).to(dev)
        x = x * torch.exp2(e)
        w = w * torch.exp2(-e) * torch.exp2(torch.arange(taps, device=dev) % 3 - 1.0)[:, None]
    if fam == "frames":
        x = x * 4.0 ** (torch.arange(NB, device=dev) % 3).float()[:, None, None, None]
    bias2 = None
    if b2:
        bias2 = rn(NB, Cout)
        if fam == "frames":
            bias2 = bias2 * 4.0 ** (torch.arange(NB, device=dev) % 3).float()[:, None]
    return x.bfloat16(), w.reshape(Cout, taps * C).bfloat16(), (0.5 * rn(Cout)).bfloat16().float(), bias2


# ------------------------------------------------------------------------------------------- CPU model of the kernel
FAULTS = ("k_tail_dropped", "a2_block_shift", "round_before_residual", "bias2_row_shift", "conv_frame_leak",
          "conv_row_wrap", "gelu_tanh")


def emulate_gemm(A, w, bias=None, bias2=None, div=1, scale=1.0, residual=None, kb1=None, geglu=False, out_f32=False,
                 fault=None):
    """The kernel's arithmetic in torch: 64-wide K blocks in order into an fp32 accumulator (K zero-padded to whole
    blocks, as the TMA unit does), fp32 epilogue (+ b, + b2[m // div], * s, + r), one rounding to bf16.  A [M, K] is
    the whole K range (split-K: concat(a, a2), kb1 = K blocks of a; convs: an im2col of conv_cols).  GEGLU: w unpacked,
    out = (v + bv) gelu(g + bg).  ``fault`` injects one bug:
      k_tail_dropped        : the last K block is skipped;
      a2_block_shift        : the A2 blocks are paired with the W block one earlier;
      round_before_residual : s (acc + b + b2) is rounded to bf16 before the residual add;
      bias2_row_shift       : bias2 row (m + 1) // div;
      gelu_tanh             : the tanh approximation of GELU.
    (The two conv faults live in conv_cols.)"""
    M, K = A.shape
    nkb = (K + KB - 1) // KB
    pad = nkb * KB - K
    Af, Wf = F.pad(A.float(), (0, pad)), F.pad(w.float(), (0, pad))
    acc = torch.zeros((M, w.shape[0]), dtype=torch.float32)
    for j in range(nkb - 1 if fault == "k_tail_dropped" else nkb):
        wj = j - 1 if fault == "a2_block_shift" and kb1 is not None and j >= kb1 else j
        acc += Af[:, j * KB:(j + 1) * KB] @ Wf[:, wj * KB:(wj + 1) * KB].t()
    if geglu:
        inner = w.shape[0] // 2
        v, gt = acc[:, :inner] + bias[:inner], acc[:, inner:] + bias[inner:]
        return (v * F.gelu(gt, approximate="tanh" if fault == "gelu_tanh" else "none")).bfloat16()
    f = acc if bias is None else acc + bias
    if bias2 is not None:
        m = torch.arange(M) + (1 if fault == "bias2_row_shift" else 0)
        f = f + bias2[(m // div).clamp(max=bias2.shape[0] - 1)]
    f = f * _f32(scale)
    if out_f32:
        return f
    if residual is not None:
        if fault == "round_before_residual":
            f = f.bfloat16().float()
        f = f + residual.float()
    return f.bfloat16()


def _cpu_cases():
    """(family, kind) pairs of the self-test; kind gemm = split-K linear with bias, bias2 (div 7) and residual; conv =
    3x3 stride 1 with bias, per-frame bias2 and residual; geglu = GEGLU GEMM."""
    return [(f, k) for f in FAMILIES[:4] for k in ("gemm", "conv")] + [(f, "geglu") for f in ("flat", "wide-gate")]


def _cpu_case(fam, kind, g):
    """-> (run(fault) -> out, ref, bnd, residual)."""
    if kind == "gemm":
        M, K1, K2, N, div = 150, 128, 72, 96, 7
        a, a2, w, b, b2, r = gemm_inputs(fam, g, M, K1, K2, N, div=div, b2_rows=(M - 1) // div + 1, residual=True)
        A = torch.cat([a, a2], 1)
        if fam == "cancel":
            r = -(gemm_ref64(A, w, b, None, b2, div, 0.75)[0]).bfloat16()
        ref, ref_abs, prod = gemm_ref64(A, w, b, None, b2, div, 0.75, r)
        run = lambda fault: emulate_gemm(A, w, b, b2, div, 0.75, r, kb1=K1 // KB, fault=fault)
        return run, ref, linear_bound(ref, ref_abs, prod, K1 + K2), r
    if kind == "conv":
        NB, H, W, C, Co = 4, 6, 5, 64, 32
        x, w, b, b2 = conv_inputs(fam, g, NB, H, W, C, Co, b2=True)
        r = torch.randn(NB * H * W, Co, generator=g).bfloat16()
        if fam == "cancel":
            r = -(conv_ref64(x, w, b, b2, H * W)[0]).bfloat16()
        ref, ref_abs, prod = conv_ref64(x, w, b, b2, H * W, 1.0, r)
        cols = lambda fault: conv_cols(x, fault=fault).reshape(NB * H * W, 9 * C)
        run = lambda fault: emulate_gemm(cols(fault), w, b, b2, H * W, 1.0, r, fault=fault)
        return run, ref, linear_bound(ref, ref_abs, prod, 9 * C), r
    a, _, w, b, _, _ = gemm_inputs(fam, g, 150, 200, 0, 128, geglu=True)
    ref, bnd = geglu_ref64(a, w, b)
    return (lambda fault: emulate_gemm(a, w, b, geglu=True, fault=fault)), ref, bnd, None


def test_bound_rejects_injected_faults():
    """The faithful model stays within the bound on every family (bf16 output rounding alone reaches a ratio of ~1, see the
    module docstring), every injected fault fails the bound or the global criterion on at least one family, and every
    family catches at least one fault."""
    caught = {f: [] for f in FAULTS}
    cases = _cpu_cases()
    for i, (fam, kind) in enumerate(cases):
        run, ref, bnd, r = _cpu_case(fam, kind, torch.Generator().manual_seed(100 + i))
        worst, rel, where = bound_check(run(None), ref, bnd, residual=r)
        print(f"faithful model {kind:5s} {fam:9s}: worst ratio {worst:.3f}, rel {rel:.2e}")
        assert worst <= 1 and rel < 5e-3, (fam, kind, where, rel)
        for fault in FAULTS:
            worst, rel, where = bound_check(run(fault), ref, bnd, residual=r)
            if worst > 1 or not rel < 5e-3:
                caught[fault].append((fam, kind, worst, rel, where))
    for fault, hits in caught.items():
        print(f"{fault:21s} rejected on " + ", ".join(f"{k}/{f} (ratio {w:.3g}, rel {r:.2e})" for f, k, w, r, _ in hits))
        if hits:
            print(f"{'':21s} first: {hits[0][4]}")
        assert hits, f"{fault} passes every family"
    for fam, kind in cases:
        assert any((fam, kind) == h[:2] for hits in caught.values() for h in hits), f"{kind} / {fam} catches no fault"


def test_cpu_references_agree():
    """conv_ref64 against F.conv2d / conv_transpose-free nearest upsampling in fp64, so the im2col orders of the reference
    are themselves checked: stride 1, stride 2 with both paddings, and the four parity classes of the folded upsample."""
    g = torch.Generator().manual_seed(5)
    NB, H, W, C, Co = 2, 6, 4, 8, 5
    x = torch.randn(NB, H, W, C, generator=g).bfloat16()
    w = torch.randn(Co, C, 3, 3, generator=g).bfloat16()
    wp = w.permute(0, 2, 3, 1).reshape(Co, 9 * C)
    xd = x.double().permute(0, 3, 1, 2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, Co)
    torch.testing.assert_close(conv_ref64(x, wp)[0], nhwc(F.conv2d(xd, w.double(), padding=1)))
    torch.testing.assert_close(conv_ref64(x, wp, kind="s2")[0], nhwc(F.conv2d(xd, w.double(), stride=2, padding=1)))
    torch.testing.assert_close(conv_ref64(x, wp, kind="s2", pad_lo=0)[0],
                               nhwc(F.conv2d(F.pad(xd, (0, 1, 0, 1)), w.double(), stride=2)))
    # the parity weights of ops.pack_upconv_weight summed in fp64 (not rounded): the four classes together are conv3x3 of
    # the nearest-2x upsampled image
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    blocks = []
    for py in (0, 1):
        for px in (0, 1):
            taps = [sum(w.double()[:, :, ky, kx] for ky in groups[py][a] for kx in groups[px][b])
                    for a in (0, 1) for b in (0, 1)]
            blocks.append(torch.stack(taps, 1).reshape(Co, -1))
    w4 = torch.cat(blocks, 0)
    up = F.interpolate(xd, scale_factor=2, mode="nearest")
    torch.testing.assert_close(conv_ref64(x, w4, kind="ups")[0], nhwc(F.conv2d(up, w.double(), padding=1)))


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture
def gemm_env():
    """gemm_env(VX_GEMM_STAGES=.., VX_GEMM_NBUF=.., VX_CONV_RR=..) sets exactly these launch switches (the others back to
    their state before the test) and makes the library re-read them; the test's end restores them all."""
    from vexpress_b200 import _ffi
    names = ("VX_GEMM_STAGES", "VX_GEMM_NBUF", "VX_CONV_RR")
    before = {n: os.environ.get(n) for n in names}

    def restore():
        for n, v in before.items():
            if v is None:
                os.environ.pop(n, None)
            else:
                os.environ[n] = v

    def switch(**kv):
        restore()
        for n, v in kv.items():
            os.environ[n] = str(v)
        _ffi.lib().vx_gemm_reload_env()

    yield switch
    restore()
    _ffi.lib().vx_gemm_reload_env()


@pytest.fixture(scope="module", autouse=True)
def _worst_ratio_summary():
    yield
    for path, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {path:16s} {worst:.3f}  ({case})")


def _sentinel_buf(shape, dtype=torch.bfloat16):
    if dtype == torch.float32:
        return torch.full(shape, _SENTINEL32, dtype=torch.int32, device="cuda").view(torch.float32)
    return torch.full(shape, _SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _bordered(rows, cols, dtype=torch.bfloat16):
    """A sentinel-filled buffer three rows taller above, five below, 8 columns wider left and 16 right (ld > cols), and
    the [rows, cols] slice inside it."""
    buf = _sentinel_buf((rows + 8, cols + 24), dtype)
    return buf, buf[3:3 + rows, 8:8 + cols]


def _in_nan(t):
    """t copied into the interior of a sentinel buffer (rows past its end, ld > its width): the view."""
    if t is None:
        return None
    buf, view = _bordered(*t.shape, t.dtype)
    view.copy_(t)
    return view


def _border_untouched(buf, inner):
    """'' or a description of the sentinel cells of ``buf`` outside the slice ``inner`` [r0:r1, c0:c1] that changed."""
    bits = buf.view(torch.int32 if buf.dtype == torch.float32 else torch.int16)
    changed = bits != (_SENTINEL32 if buf.dtype == torch.float32 else _SENTINEL)
    changed[inner] = False
    n = int(changed.sum())
    return "" if n == 0 else f"{n} cells outside the output slice written, first at {changed.nonzero()[0].tolist()}"


_INNER = (slice(3, -5), slice(8, -16))


def _judge(path, case, fam, out, ref, bnd, border="", bf16_out=True, residual=None):
    """Bound, global criterion, NaN inside and sentinels outside the output -> '' or a failure message."""
    torch.cuda.synchronize()
    worst, rel, where = bound_check(out, ref, bnd, bf16_out, residual)
    print(f"{path:16s} {case} {fam:9s}: worst ratio {worst:.3f}, rel {rel:.2e}")
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


def _seed(*ints):
    s = 0
    for i in ints:
        s = (s * 1000003 + int(i)) % (1 << 31)
    return s


def _run_gemm(ops, fams, M, K1, N, *, K2=0, bias=True, div=0, scale=1.0, residual=False, out_f32=False, block_n=0,
              geglu=False, path=None):
    """ops.gemm over each family with a / a2 / w / residual as interior views of sentinel buffers and out inside a
    sentinel border -> {family: output copy}."""
    path = path or ("GEGLU" if geglu else "fp32 out" if out_f32 else "split-K" if K2 else "plain")
    case = (f"M {M} K {K1}{'+%d' % K2 if K2 else ''} N {N} bias {int(bias)} div {div} scale {scale} "
            f"res {int(residual)} bn {block_n}")
    fails, outs = [], {}
    for fam in fams:
        g = torch.Generator(device="cuda").manual_seed(_seed(M, K1, K2, N, div, block_n, FAMILIES.index(fam)))
        b2_rows = (M - 1) // div + 1 if div else 0
        a, a2, w, b, b2, r = gemm_inputs(fam, g, M, K1, K2, N, div=div or 128, b2_rows=b2_rows, residual=residual,
                                         geglu=geglu)
        b = b if bias or geglu else None
        dtype = torch.float32 if out_f32 else torch.bfloat16
        if geglu:
            wp, bp, _ = ops.pack_geglu(w, b)
            obuf, out = _bordered(M, N // 2)
            ops.gemm(_in_nan(a), _in_nan(wp), bp, geglu=True, out=out)
            ref, bnd = geglu_ref64(a, w, b)
        else:
            if fam == "cancel" and residual:
                r = -(gemm_ref64(a, w, b, a2, b2, div or 1, scale)[0]).bfloat16()
            obuf, out = _bordered(M, N, dtype)
            ops.gemm(_in_nan(a), _in_nan(w), b, a2=_in_nan(a2), bias2=b2, bias2_div=div or 1, scale=scale,
                     residual=_in_nan(r), out=out, block_n=block_n, out_f32=out_f32)
            ref, ref_abs, prod = gemm_ref64(a, w, b, a2, b2, div or 1, scale, r)
            bnd = linear_bound(ref, ref_abs, prod, K1 + K2)
        fails.append(_judge(path, case, fam, out, ref, bnd, _border_untouched(obuf, _INNER), not out_f32, r))
        outs[fam] = out.clone()
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)
    return outs


def _pick_block_n(tiles_m, N, gran, total_kb):
    """vx_gemm.cu pick_block_n: the wgmma N the library chooses."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    best, best_cost = 0, 1e30
    for bn in range(256, gran - 1, -gran):
        if N % bn or bn not in (16, 32, 64, 96, 128, 160, 192, 256):
            continue
        waves = (tiles_m * (N // bn) + sms - 1) // sms
        cost = waves * (total_kb * (max(4.0 * bn, 128.0 + 2.0 * bn) + 40.0) + 4.0 * bn)
        if cost < best_cost * 0.999:
            best, best_cost = bn, cost
    return best


def _conv_tile(NB, H, W):
    """vx_gemm.cu conv3x3_entry: (wbox, hbox, nbox) of the pixel rectangle one 128-row tile covers."""
    if W >= 128:
        wbox = 128
        while W % wbox:
            wbox -= 1
        return wbox, 1, 1
    hbox, nbox = 128 // W, 1
    if hbox > H:
        hbox = H
        nbox = max(1, min(NB, 128 // (W * H)))
        while NB % nbox:
            nbox -= 1
    else:
        while H % hbox:
            hbox -= 1
    return W, hbox, nbox


def _conv_path(NB, H, W, C, Cout, block_n=0, rr=True):
    """'conv row-reuse' when the stride-1 conv takes the row-reuse producer (one A box of hbox + 2 image rows serves the
    three dy taps), else 'conv tap by tap'."""
    wbox, hbox, nbox = _conv_tile(NB, H, W)
    rows = wbox * hbox * nbox
    if rr and nbox == 1 and wbox == W and hbox >= 2 and rows == 128 and W % 8 == 0:
        bn = block_n or _pick_block_n(NB * H * W // rows, Cout, 32, 9 * (C // KB))
        st = (hbox + 2) * W * KB * 2 + 3 * bn * KB * 2
        if 2 * st + bn // 32 * 8192 <= 227 * 1024 - 2048:
            return "conv row-reuse"
    return "conv tap by tap"


def _run_conv(ops, fams, NB, H, W, C, Cout, *, kind="s1", pad_lo=1, epilogue=True, scale=1.0, block_n=0, rr=True):
    """conv3x3 (kind s1, with bias, per-frame bias2, scale and an interior-view residual when ``epilogue``), conv3x3_s2
    (kind s2) or upconv3x3 (kind ups) over each family.  The input is frames 1..NB of a buffer whose frames 0 and NB + 1
    are NaN; out sits inside a sentinel border -> {family: output copy}."""
    path = {"s1": _conv_path(NB, H, W, C, Cout, block_n, rr), "s2": "stride 2", "ups": "ups"}[kind]
    Ho, Wo = (H // 2, W // 2) if kind == "s2" else (H, W)
    rows = NB * Ho * Wo * (4 if kind == "ups" else 1)
    case = f"NB {NB} {H}x{W} C {C}->{Cout}" + (f" pad_lo {pad_lo}" if kind == "s2" else "") + (f" bn {block_n}" if block_n else "")
    with_epi = epilogue and kind == "s1"
    fails, outs = [], {}
    for fam in fams:
        if fam == "cancel" and not with_epi:
            continue
        g = torch.Generator(device="cuda").manual_seed(_seed(NB, H, W, C, Cout, pad_lo, FAMILIES.index(fam)))
        taps = 4 if kind == "ups" else 9
        x, w, b, b2 = conv_inputs(fam, g, NB, H, W, C, Cout * (4 if kind == "ups" else 1), taps, b2=with_epi)
        b = b[:Cout].contiguous()
        xb = _sentinel_buf((NB + 2, H, W, C))
        xb[1:NB + 1] = x
        xv = xb[1:NB + 1]
        obuf, out = _bordered(rows, Cout)
        r = None
        if kind == "s1":
            div = H * W
            if with_epi:
                r = (-(conv_ref64(x, w, b, b2, div, scale)[0]).bfloat16() if fam == "cancel"
                     else torch.randn(rows, Cout, device="cuda", generator=g).bfloat16())
            ops.conv3x3(xv, w, b, bias2=b2, bias2_div=div, scale=scale, residual=_in_nan(r), out=out, block_n=block_n)
            ref, ref_abs, prod = conv_ref64(x, w, b, b2, div, scale, r)
        elif kind == "s2":
            ops.conv3x3_s2(xv, w, b, pad_lo=pad_lo, out=out, block_n=block_n)
            ref, ref_abs, prod = conv_ref64(x, w, b, kind="s2", pad_lo=pad_lo)
        else:
            ops.upconv3x3(xv, w, b, out=out, block_n=block_n)
            ref, ref_abs, prod = conv_ref64(x, w, b, kind="ups")
        bnd = linear_bound(ref, ref_abs, prod, w.shape[1])
        fails.append(_judge(path, case, fam, out, ref, bnd, _border_untouched(obuf, _INNER), True, r))
        outs[fam] = out.clone()
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)
    return outs


LINEAR = ("flat", "blocks", "cancel", "frames")
SHORT = ("flat", "blocks")


# ---- plain GEMM: row tails (one row, a partial tile, exactly one tile, one row past it, more tiles than SMs plus a
# one-row tail) and K tails (K < 64, K % 64 != 0, 7 K blocks against a 6-stage ring, long K loops)
@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 7, 127, 128, 129, 300, 128 * 133 + 1])
def test_gemm_rows_within_bound(ops, M):
    _run_gemm(ops, LINEAR, M, 448, 320, div=7, scale=-1.5, residual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 56, 64, 72, 200, 320, 448, 1280, 5120])
def test_gemm_k_within_bound(ops, K):
    _run_gemm(ops, LINEAR, 300, K, 96, residual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("bias,div,scale,residual", [
    (True, 0, 1.0, False), (False, 0, 1.0, False), (True, 1, 1.0, False), (True, 7, 1.0, False), (True, 128, 1.0, False),
    (True, 129, 1.0, False), (True, 300, 1.0, False), (True, 0, 0.37, False), (True, 0, -1.5, True), (False, 129, 0.37, True)])
def test_gemm_epilogue_within_bound(ops, bias, div, scale, residual):
    _run_gemm(ops, LINEAR if residual else ("flat", "blocks", "frames"), 300, 200, 128, bias=bias, div=div, scale=scale,
              residual=residual)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [32, 64, 96, 128, 160, 192, 256])
def test_gemm_every_block_n_within_bound(ops, block_n):
    """N = 3840 divides by every supported column-tile width."""
    _run_gemm(ops, ("flat", "cancel"), 300, 200, 3840, div=129, residual=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [16, 0])
@pytest.mark.parametrize("N", [16, 48, 80, 208])
def test_gemm_fp32_out_within_bound(ops, N, block_n):
    """fp32 output (the attention-score form), N = 16 x odd, with bias2 and a scale: the accumulator itself is checked."""
    _run_gemm(ops, ("flat", "blocks", "frames"), 300, 200, N, div=7, scale=0.125, out_f32=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("K2", [8, 72, 320, 1280])
@pytest.mark.parametrize("K1", [64, 320, 1280])
def test_gemm_split_k_within_bound(ops, K1, K2):
    """K over two sources (concat(a, a2) folded into the K loop): the A / A2 boundary and the A2 tail."""
    _run_gemm(ops, LINEAR, 300, K1, 160, K2=K2, residual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [512, 384, 192])
def test_gemm_geglu_within_bound(ops, N):
    """One N per geglu_block_n (256 / 128 / 64 accumulator columns per tile), through the pack_geglu round trip."""
    _run_gemm(ops, ("flat", "blocks", "frames", "wide-gate"), 300, 320, N, geglu=True)


# ---- 3x3 convolution, stride 1
CONV_S1 = [
    (2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 1280, 1280), (4, 8, 8, 1280, 1280),   # 512: rr hbox 2/4/8, nbox
    (1, 96, 96, 320, 320), (2, 48, 48, 640, 640), (2, 24, 24, 1280, 1280), (4, 12, 12, 1280, 1280),  # configs[4]
    (3, 16, 24, 128, 128), (2, 8, 24, 320, 320),                                                    # non-square
    (2, 16, 16, 64, 64), (2, 32, 32, 960, 640), (2, 16, 16, 1920, 1280), (2, 8, 8, 2560, 1280)]      # channel counts
CONV_VAE = [(1, 128, 128, 512, 512), (1, 192, 192, 512, 512), (1, 256, 256, 256, 256), (1, 384, 384, 256, 256),
            (1, 512, 512, 128, 128), (1, 768, 768, 128, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout", CONV_S1)
def test_conv3x3_within_bound(ops, NB, H, W, C, Cout):
    _run_conv(ops, LINEAR, NB, H, W, C, Cout, scale=0.875)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout", CONV_VAE)
def test_conv3x3_vae_within_bound(ops, NB, H, W, C, Cout):
    """The VAE levels: one frame, W >= 128 (wbox 128, or 96 at the 192-wide level)."""
    _run_conv(ops, SHORT, NB, H, W, C, Cout, epilogue=False)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout", [c for c in CONV_S1 if c[1:3] in ((64, 64), (32, 32), (16, 16))])
def test_conv3x3_tap_by_tap_within_bound(ops, gemm_env, NB, H, W, C, Cout):
    """The row-reuse shapes again with row reuse off (VX_CONV_RR=0): the taps run one by one and sum in another order,
    so the two paths are held to the bound, not to each other."""
    gemm_env(VX_CONV_RR=0)
    _run_conv(ops, ("flat", "blocks", "frames"), NB, H, W, C, Cout, scale=0.875, rr=False)


# ---- stride 2 and the folded upsample
@pytest.mark.gpu
@pytest.mark.parametrize("pad_lo", [1, 0])
@pytest.mark.parametrize("NB,H,W,C,Cout", [
    (2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 1280, 1280), (1, 96, 96, 320, 320), (2, 48, 48, 640, 640),
    (2, 24, 24, 1280, 1280), (1, 512, 512, 128, 128), (1, 256, 256, 256, 256), (1, 768, 768, 128, 128)])
def test_conv3x3_s2_within_bound(ops, NB, H, W, C, Cout, pad_lo):
    _run_conv(ops, ("flat", "blocks", "frames"), NB, H, W, C, Cout, kind="s2", pad_lo=pad_lo)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout", [
    (2, 8, 8, 1280, 1280), (2, 16, 16, 1280, 1280), (2, 32, 32, 640, 640), (2, 12, 12, 1280, 1280),
    (2, 24, 24, 1280, 1280), (1, 48, 48, 640, 640), (1, 64, 64, 512, 512), (1, 96, 96, 512, 512),
    (1, 128, 128, 512, 512), (1, 192, 192, 512, 512), (1, 256, 256, 256, 256), (1, 384, 384, 256, 256)])
def test_upconv3x3_within_bound(ops, NB, H, W, C, Cout):
    """conv3x3(upsample2x(x)) as four parity-class 2x2 convolutions, UNet 8 -> 16 ... 48 -> 96 and VAE 64 -> 128 ...
    384 -> 768 (inputs 96 and more pixels wide: wbox 96 / 128, hbox 1)."""
    _run_conv(ops, ("flat", "blocks", "frames") if H * W <= 4096 else SHORT, NB, H, W, C, Cout, kind="ups")


# ---- ring depth and staging count: no arithmetic changes, so bit-identical to the default launch
@pytest.mark.gpu
@pytest.mark.parametrize("knob,value", [("VX_GEMM_STAGES", 2), ("VX_GEMM_STAGES", 3), ("VX_GEMM_STAGES", 7),
                                        ("VX_GEMM_NBUF", 1), ("VX_GEMM_NBUF", 2)])
@pytest.mark.parametrize("kind", ["gemm", "conv tap by tap", "conv row-reuse"])
def test_stages_and_staging_bit_identical(ops, gemm_env, kind, knob, value):
    """Every case has more tiles than SMs.  Row reuse picks its own ring depth, so VX_GEMM_STAGES does not apply to it."""
    if kind == "conv row-reuse" and knob == "VX_GEMM_STAGES":
        pytest.skip("row reuse ignores VX_GEMM_STAGES")
    if kind == "gemm":
        run = lambda: _run_gemm(ops, ("flat", "cancel"), 128 * 133 + 1, 448, 320, div=7, residual=True)
    else:
        shape = (4, 48, 48, 320, 320) if kind == "conv tap by tap" else (4, 64, 64, 320, 320)
        assert _conv_path(*shape) == kind
        run = lambda: _run_conv(ops, ("flat", "cancel"), *shape)
    gemm_env()
    base = run()
    gemm_env(**{knob: value})
    forced = run()
    for fam in base:
        assert torch.equal(base[fam], forced[fam]), f"{kind} {knob}={value} {fam}: differs from the default launch"


# ---- production calls, exactly as the model makes them
def _temb_slice(g, NB, Cout):
    """The time embedding of the whole UNet ([2 CFG rows, all blocks' channels], fp32) and the block's column slice."""
    temb = torch.randn(2, 3 * Cout, device="cuda", generator=g)
    return temb[:, Cout:2 * Cout]


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,C", [(32, 64, 320), (32, 8, 1280)])
def test_resnet_convs_production_within_bound(ops, NB, H, C):
    """conv1 with bias2 = a strided column slice of temb read through bias2_div = NB H W (row 0 serves every row), conv2
    with residual = the block input."""
    g = torch.Generator(device="cuda").manual_seed(_seed(NB, H, C))
    x, w, b, _ = conv_inputs("flat", g, NB, H, H, C, C)
    t = _temb_slice(g, NB, C)
    div = NB * H * H
    h = ops.conv3x3(x, w, b, bias2=t, bias2_div=div)
    ref, ref_abs, prod = conv_ref64(x, w, b, t, div)
    msg = [_judge(_conv_path(NB, H, H, C, C), f"resnet conv1 NB {NB} {H}x{H} C {C}", "given", h, ref,
                  linear_bound(ref, ref_abs, prod, 9 * C))]
    sc = torch.randn(NB * H * H, C, device="cuda", generator=g).bfloat16()
    o = ops.conv3x3(x, w, b, residual=sc)
    ref, ref_abs, prod = conv_ref64(x, w, b, residual=sc)
    msg.append(_judge(_conv_path(NB, H, H, C, C), f"resnet conv2 NB {NB} {H}x{H} C {C}", "given", o, ref,
                      linear_bound(ref, ref_abs, prod, 9 * C), residual=sc))
    msg = [m for m in msg if m]
    assert not msg, "\n".join(msg)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K1,K2,N", [(131072, 640, 320, 320), (8192, 1280, 640, 640)])
def test_conv_shortcut_production_within_bound(ops, M, K1, K2, N):
    """The up blocks' 1x1 shortcut over concat(h, skip), contiguous operands."""
    g = torch.Generator(device="cuda").manual_seed(_seed(M, K1, K2))
    a, a2, w, b, _, _ = gemm_inputs("flat", g, M, K1, K2, N)
    a, a2 = a.contiguous(), a2.contiguous()
    out = ops.gemm(a, w, b, a2=a2)
    ref, ref_abs, prod = gemm_ref64(a, w, b, a2)
    m = _judge("split-K", f"conv_shortcut M {M} K {K1}+{K2} N {N}", "given", out, ref, linear_bound(ref, ref_abs, prod, K1 + K2))
    assert not m, m


@pytest.mark.gpu
@pytest.mark.parametrize("M,C", [(131072, 320), (2048, 1280)])
def test_feedforward_production_within_bound(ops, M, C):
    """FF1 (C -> 8 C accumulator columns, GEGLU in the epilogue -> 4 C) and FF2 (4 C -> C with the residual) at the 64 x 64
    and 8 x 8 levels of a 2 x 16-frame window."""
    g = torch.Generator(device="cuda").manual_seed(_seed(M, C))
    n, _, w1, b1, _, _ = gemm_inputs("flat", g, M, C, 0, 8 * C, geglu=True)
    wp, bp, _ = ops.pack_geglu(w1, b1)
    h = ops.gemm(n, wp, bp, geglu=True)
    ref, bnd = geglu_ref64(n, w1, b1)
    msg = [_judge("GEGLU", f"FF1 M {M} {C} -> {8 * C}", "given", h, ref, bnd)]
    _, _, w2, b2, _, _ = gemm_inputs("flat", g, M, 4 * C, 0, C)
    res = torch.randn(M, C, device="cuda", generator=g).bfloat16()
    o = ops.gemm(h, w2, b2, residual=res)
    ref, ref_abs, prod = gemm_ref64(h, w2, b2, residual=res)
    msg.append(_judge("plain", f"FF2 M {M} {4 * C} -> {C}", "given", o, ref, linear_bound(ref, ref_abs, prod, 4 * C),
                      residual=res))
    msg = [m for m in msg if m]
    assert not msg, "\n".join(msg)


@pytest.mark.gpu
@pytest.mark.parametrize("HW", [4096, 9216])
def test_vae_attention_production_within_bound(ops, HW):
    """The VAE mid-block attention of one frame at 64 x 64 and 96 x 96 latents (vae.py _attn): fp32 scores into ``out=``
    with scale C^-1/2, V^T = Wv xn^T (the activations as the W operand), and P V + bv into a row slice of o (K = HW)."""
    C = 512
    g = torch.Generator(device="cuda").manual_seed(HW)
    q, k, xn = (torch.randn(2 * HW, C, device="cuda", generator=g).bfloat16() for _ in range(3))
    sl = slice(HW, 2 * HW)
    scores = torch.empty((HW, HW), device="cuda", dtype=torch.float32)
    ops.gemm(q[sl], k[sl], scale=C ** -0.5, out=scores, out_f32=True)
    ref, ref_abs, prod = gemm_ref64(q[sl], k[sl], scale=C ** -0.5)
    msg = [_judge("fp32 out", f"VAE scores HW {HW}", "given", scores, ref, linear_bound(ref, ref_abs, prod, C),
                  bf16_out=False)]
    del ref, ref_abs, prod
    wv = (torch.randn(C, C, device="cuda", generator=g) / math.sqrt(C)).bfloat16()
    vt = torch.empty((C, HW), device="cuda", dtype=torch.bfloat16)
    ops.gemm(wv, xn[sl], out=vt)
    ref, ref_abs, prod = gemm_ref64(wv, xn[sl])
    msg.append(_judge("plain", f"VAE V^T HW {HW}", "given", vt, ref, linear_bound(ref, ref_abs, prod, C)))
    probs = torch.softmax(3 * torch.randn(HW, HW, device="cuda", generator=g), -1).bfloat16()
    bv = torch.randn(C, device="cuda", generator=g).bfloat16().float()
    o = torch.full((2 * HW, C), float("nan"), device="cuda", dtype=torch.bfloat16)
    ops.gemm(probs, vt, bv, out=o[sl])
    ref, ref_abs, prod = gemm_ref64(probs, vt, bv)
    msg.append(_judge("plain", f"VAE P V HW {HW}", "given", o[sl], ref, linear_bound(ref, ref_abs, prod, HW)))
    if not torch.isnan(o[:HW].float()).all():
        msg.append("P V wrote outside its row slice")
    msg = [m for m in msg if m]
    assert not msg, "\n".join(msg)


# ---- conv_out_tc: the conv on the GEMM kernel (Cout zero-padded to 32) and vx_extract_planar
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unet", "vae", "encoder"])
def test_conv_out_tc_within_bound(ops, which):
    """UNet 320 -> 4 (bf16 planar), VAE 128 -> 3 with post = (v / 2 + 0.5).clamp(0, 1) into the fp32 (3, L, H, W) video
    view the pipeline passes (frames outside the view hold the sentinel), encoder mean 512 -> 4 (bf16)."""
    NB, H, C, co, L, post, dtype = {"unet": (4, 64, 320, 4, 4, False, torch.bfloat16),
                                    "vae": (2, 128, 128, 3, 4, True, torch.float32),
                                    "encoder": (1, 64, 512, 4, 1, False, torch.bfloat16)}[which]
    fails = []
    for fam in ("flat", "blocks", "frames"):
        g = torch.Generator(device="cuda").manual_seed(_seed(NB, H, C, FAMILIES.index(fam)))
        x, w, _, _ = conv_inputs(fam, g, NB, H, H, C, co)
        b = torch.randn(co, device="cuda", generator=g).bfloat16().float()
        wp, bp = ops.pack_conv_out(w.view(co, 3, 3, C).permute(0, 3, 1, 2), b)
        video = _sentinel_buf((co, L + 2, H, H), dtype)
        out = video[:, 1:NB + 1].permute(1, 0, 2, 3)
        ops.conv_out_tc(x.view(NB * H * H, C), NB, H, H, wp, bp, out, post=post)
        ref, ref_abs, prod = conv_ref64(x, wp, bp)
        ref = ref[:, :co]
        bnd = 2.0 ** -8 * ref.abs() + linear_bound(ref, ref_abs[:, :co], prod[:, :co], 9 * C)   # conv output in bf16
        if post:
            ref, bnd = (0.5 * ref + 0.5).clamp(0, 1), 0.5 * bnd + 2.0 ** -22
        got = out.permute(0, 2, 3, 1).reshape(-1, co)
        rest = torch.cat([video[:, :1], video[:, NB + 1:]], 1)
        ok = (rest.view(torch.int32 if dtype == torch.float32 else torch.int16)
              == (_SENTINEL32 if dtype == torch.float32 else _SENTINEL)).all()
        fails.append(_judge("conv_out_tc", f"{which} NB {NB} {H}x{H} C {C}->{co} post {int(post)}", fam, got, ref, bnd,
                            "" if ok else "frames outside the output view written", dtype == torch.bfloat16 and post))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


# ---- conv_in: fp32 CUDA-core 3x3 from 4 planar channels
def _conv_in_ref64(x, w, bias, addend=None, add_frame=None, pre=None):
    """(ref, bound without the output rounding) [NB H W, Cout] of vx_conv_in.  x planar bf16 (NB, 4, H, W), w fp32 (Cout,
    4, 3, 3).  pre = (scale, pre_w, pre_b): the kernel's per-pixel v -> bf16(pre_w bf16(scale v) + pre_b); bf16(scale v)
    is reproduced exactly (one fp32 product, then round to nearest even), the second rounding in fp64 -- where the fp32
    sum the kernel rounds can fall on the other side of a bf16 rounding boundary, the bound admits the neighbouring
    value (|W| conv |v_hi - v_lo|)."""
    NB, _, H, W = x.shape
    v = x.double()
    amb = None
    if pre is not None:
        s, pw, pb = pre
        t = (x.float() * _f32(s)).bfloat16().double()
        a = torch.einsum("ck,nkhw->nchw", pw.double(), t) + pb.double()[None, :, None, None]
        e = 2.0 ** -21 * (torch.einsum("ck,nkhw->nchw", pw.double().abs(), t.abs()) + pb.double().abs()[None, :, None, None])
        rnd = lambda z: z.float().bfloat16().double()
        v, amb = rnd(a), (rnd(a + e) - rnd(a - e)).abs()
    wd = w.double()
    ref = F.conv2d(v, wd, bias.double(), padding=1)
    ref_abs = F.conv2d(v.abs(), wd.abs(), bias.double().abs(), padding=1)
    prod = F.conv2d(v.abs(), wd.abs(), padding=1)
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(NB * H * W, -1)
    ref, ref_abs, prod = nhwc(ref), nhwc(ref_abs), nhwc(prod)
    if addend is not None:
        rows = (add_frame.long()[:, None] * (H * W) + torch.arange(H * W, device=x.device)[None]).reshape(-1)
        ad = addend[rows].double()
        ref, ref_abs = ref + ad, ref_abs + ad.abs()
    bnd = linear_bound(ref, ref_abs, prod, 36)
    if amb is not None:
        bnd = bnd + nhwc(F.conv2d(amb, wd.abs(), padding=1))
    return ref, bnd


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unet", "vae"])
def test_conv_in_within_bound(ops, which):
    """UNet 4 -> 320 on a (frames, 4, H, W) view of a (4, frames, H, W) tensor with the kps addend gathered per frame by
    add_frame; the VAE decoder form 4 -> 512 with pre_scale = 1 / 0.18215 and the 4 x 4 post_quant_conv."""
    NB, H, Cout = (6, 64, 320) if which == "unet" else (2, 96, 512)
    fails = []
    for fam in ("flat", "frames"):
        g = torch.Generator(device="cuda").manual_seed(_seed(NB, H, Cout, FAMILIES.index(fam)))
        rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
        x = rn(4, NB, H, H)
        if fam == "frames":
            x = x * 4.0 ** (torch.arange(NB, device="cuda") % 3).float()[None, :, None, None]
        x = x.bfloat16().permute(1, 0, 2, 3)
        w = (rn(Cout, 4, 3, 3) / 6).bfloat16().float()
        b = rn(Cout).bfloat16().float()
        addend = add_frame = pre = None
        kw = {}
        if which == "unet":
            addend = rn(3 * H * H, Cout).bfloat16()
            add_frame = torch.tensor([(2 - n) % 3 for n in range(NB)], device="cuda", dtype=torch.int32)
            kw = dict(addend=addend, add_frame=add_frame)
        else:
            pre = (1 / 0.18215, rn(4, 4).bfloat16().float(), rn(4).bfloat16().float())
            kw = dict(pre_scale=pre[0], pre_w=pre[1], pre_b=pre[2])
        obuf, out = _bordered(NB * H * H, Cout)
        ops.conv_in(x, w.reshape(Cout, 36).t().contiguous(), b, Cout, out=out, **kw)
        ref, bnd = _conv_in_ref64(x, w, b, addend, add_frame, pre)
        fails.append(_judge("conv_in", f"{which} NB {NB} {H}x{H} 4->{Cout}", fam, out, ref, bnd,
                            _border_untouched(obuf, _INNER)))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


# ---- the wrappers check bias / bias2 before they hand raw pointers to the kernel
@pytest.mark.gpu
def test_bias_arguments_are_validated(ops):
    dev = "cuda"
    M, K, N = 300, 64, 96
    a = torch.randn(M, K, device=dev).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    b = torch.randn(N, device=dev)
    wide = torch.randn(M, 3 * N, device=dev)
    bad = {
        "bf16 bias": dict(bias=b.bfloat16()),
        "bias on the host": dict(bias=b.cpu()),
        "bias too short": dict(bias=b[:N - 2]),
        "strided bias": dict(bias=torch.randn(2 * N, device=dev)[::2]),
        "bf16 bias2": dict(bias2=wide[:, :N].contiguous().bfloat16()),
        "bias2 too few rows": dict(bias2=wide[:M // 7, :N].contiguous(), bias2_div=7),
        "bias2 wrong width": dict(bias2=wide[:, :N + 4].contiguous()),
        "bias2 column slice read at every row": dict(bias2=wide[:, N:2 * N]),
        "bias2 column slice read at two rows": dict(bias2=wide[:, N:2 * N], bias2_div=M - 1),
        "bias2_div 0": dict(bias2=wide[:, :N].contiguous(), bias2_div=0),
        "misaligned bias2": dict(bias2=wide.reshape(-1)[1:1 + M * N].view(M, N)),
    }
    for what, kw in bad.items():
        with pytest.raises(ValueError):
            ops.gemm(a, w, **{"bias": b, **kw})
        print(f"ops.gemm rejects: {what}")
    x = torch.randn(2, 8, 8, 64, device=dev).bfloat16()
    wc = torch.randn(N, 9 * 64, device=dev).bfloat16()
    with pytest.raises(ValueError):
        ops.conv3x3(x, wc, b, bias2=wide[:1, :N].contiguous(), bias2_div=64)      # two frames, one row
    with pytest.raises(ValueError):
        ops.conv3x3_s2(x, wc, b.bfloat16())
    with pytest.raises(ValueError):
        ops.upconv3x3(x, torch.randn(4 * N, 4 * 64, device=dev).bfloat16(), b[:N // 2])
    # accepted: the production form, a strided column slice of which only row 0 is read
    g = torch.Generator(device=dev).manual_seed(3)
    a, _, w, b, _, _ = gemm_inputs("flat", g, M, K, 0, N)
    t = _temb_slice(g, 1, N)
    out = ops.gemm(a, w, b, bias2=t, bias2_div=M)
    ref, ref_abs, prod = gemm_ref64(a, w, b, bias2=t, div=M)
    m = _judge("plain", "temb slice, div = M", "given", out, ref, linear_bound(ref, ref_abs, prod, K))
    assert not m, m
