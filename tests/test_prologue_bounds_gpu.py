"""The conditioning prologue (``modules/prologue.py``: VKpsGuider and AudioProjection) against fp64 references at the
shapes the pipeline runs: every kernel call of a real forward judged element by element, the gather kernel on its own,
the modules against their fp64 oracle (the perceiver one residual branch at a time), batching and chunking invariants,
and the two pipeline hooks that call them.

The prologue runs once per video, but its outputs condition every UNet forward of every step (the kps features are
conv_in's addend of every frame, the audio tokens the K / V of every audio cross-attention at weight 3.0), so an error
here is applied at every step rather than averaged away by the sampler.

1. Every kernel call (``_Recorder``).  ``prologue.ops`` is replaced by a proxy that forwards each call to the real ops,
   then judges its output at once against an fp64 reference of exactly the operands the kernel read, and lets it go
   (the 768^2 first-layer columns alone are 2.7 GB in bf16):
     conv_in     ``_conv_in_ref64`` (tests/test_gemm_bounds_gpu.py);
     im2col3x3   the gather must be bit-exact, and each gathered SiLU value within the bound below;
     gemm        ``linear_ref64`` + ``linear_bound`` on the columns and packed weights the kernel read; GELU through the
                 GEGLU epilogue: ``geglu_ref64`` on the unpacked [0 | w1] weights with bias [1 | 0];
     layernorm   ``layernorm_ref64`` (tests/test_norm_bounds_gpu.py);
     attention   ``attention_ref64`` (tests/test_attention_bounds_gpu.py) on the strided K / V column halves of to_kv.
   Each keeps the global criterion of its home file (relative L2 < 5e-3, attention 4e-3).  The guider's channel counts
   are zero-padded to multiples of 32: the padded columns of every layer's output (16..31 of conv_in and blocks.0) must
   be exactly 0 -- the next layer's zero weight columns hide any other value until it is Inf, and then it is NaN.

   SiLU in the gather: the kernel computes v = x / (1 + __expf(-x)) in fp32 (IEEE division: the library is built
   without fast math) and rounds v to bf16.  __expf(-x) is within 2 + 1.173 |x| ulp (CUDA C Programming Guide), a
   relative (2 + 1.173 |x|) 2^-23; 1 + e and the division round once each (2^-24 each); an error of relative d in e
   moves 1 / (1 + e) by at most relative d.  So |v - silu(x)| <= (3 + 1.173 |x|) 2^-23 |silu(x)|, which the term
   e_act(x) = (5 + 1.2 |x|) 2^-23 |silu(x)| + 2^-126 of ``_act_terms`` covers (the same form as the skinny linear's SiLU);
   below x = -88, __expf overflows and v = -0 while |silu(x)| < 2^-122: e_act allows all of |silu(x)| there.  The bf16
   rounding adds 2^-8 |ref| (``bound_check``).  A SiLU rounded twice, bf16(x bf16(sigmoid(x))), exceeds it
   (``test_silu_bound_self_test``).

2. ``im2col3x3`` on its own: strides 1 and 2, pad_lo 1 and 0 (the VAE encoder's Downsample2D), odd H / W at stride 2,
   C = 32 and 96 (the guider's widths), inputs the inner frames of a buffer whose first and last frames are NaN, output
   into a sentinel-bordered buffer through ``out=``.

3. Modules against fp64, with the rule of tests/test_blocks_gpu.py: e_prod = ||out - ref64|| / ||B||, e_eager the same
   measure of the oracle run in torch.bfloat16 on the GPU (the reference's own arithmetic on its device); a case passes
   when e_prod <= min(max(1.5 e_eager, FLOOR), CEIL) and the output is finite.
   AudioProjection, one branch at a time: for layer i and branch attn (layers.i.0.to_out) or ff (layers.i.1.3), every
   other layer's to_out and .3 weights are zeroed, so the latents pass through them unchanged and the live branch is
   teacher-forced on exact inputs through the real module.  B = ref64 - ref64(live branch zeroed too); the branch is
   scaled by a power of two until B carries at least MIN_SHARE of the output (||B|| / ||ref64||, asserted on the fp64
   data).  Also the unmodified module at L = 300 (B = its whole output) and the proj_in -> proj_out -> norm_out path
   with every branch zeroed.  VKpsGuider (no residual: B = the whole output) at 512^2, t = 16, b = 1 and 2, and 768^2,
   t = 8; input families v-kps (the reference's draw_v_kps_image: black canvas, two sticks of half-width 4 at 0.6, three
   radius-4 dots in R / G / B, moving from frame to frame), dense uniform noise, and all-black frames, where every
   interior output pixel must be bitwise equal to every other at every layer (equal im2col rows give equal GEMM bits).
   Audio families: wav2vec-like states (per-channel scaled normals) through ``audio_frame_windows`` (the first and last
   two frames hold zero rows), and windows that differ strongly from frame to frame.
   The synthetic state dict (``O.synth_state_dict``) gives pos_emb rows of std 0.036 and LayerNorm weights 1 +- 0.02,
   which no trained checkpoint has: ``_proj_sd`` redraws pos_emb at std 0.5 and the LayerNorm scales / shifts as
   1 + 0.25 N(0, 1) / 0.1 N(0, 1), so that a shifted pos_emb row or swapped norms change the output visibly.

4. Batching and chunking, bit-exact: the guider's frame j does not depend on frames_per_chunk, its place in the chunk
   or b; ``prepare_kps_feature`` equals the per-frame guider outputs (uncond half exactly 0), also from HWC uint8
   arrays; AudioProjection frame l at L = 300 equals the L = 1 call on window l.

5. Fault catalogue (CPU): each fault is emulated in an fp64 model (``guider64`` / ``proj64``, equal to the oracle when
   no fault is set) and must move the measure of at least one case by 2x that case's threshold.  GELU with the tanh
   form is a kernel fault the module measure cannot see (gelu_tanh - gelu_erf < 1e-3): it is checked where the
   recorder sees it, against the GEGLU call's elementwise bound.  Fault size / threshold (the case that shows it
   most), CPU, guider 64^2 x 4 frames in chunks of 2, projection L = 6:
       no SiLU after conv_in            2.18e-1 / 1.00e-2     pos_emb rows shifted by one      3.85e-1 / 1.00e-2
       SiLU after conv_out              5.01e-1 / 1.00e-2     attention scale 1 / hd           5.16e-1 / 1.00e-2
       stride 2 on the same-width conv  1.73e-1 / 1.00e-2     K / V from x only                7.02e-1 / 1.35e-2
       stride-2 padding (0, 1, 0, 1)    1.96e-1 / 1.00e-2     K and V halves swapped           1.05    / 1.00e-2
       im2col K order (channel, tap)    7.58e-1 / 1.00e-2     norm1 and norm2 swapped          5.90e-1 / 1.35e-2
       a frame across a chunk boundary  7.53e-2 / 1.00e-2     frame l reads window l + 1       8.29e-1 / 1.00e-2
       conv_out bias dropped            8.99e-1 / 1.00e-2     norm_out dropped                 9.76e-1 / 1.00e-2
       tanh-GELU: worst GEGLU bound ratio 9.7 (the erf form 0.68)
   The smallest margin is 7.5x (a frame moved across a chunk boundary: neighbouring v-kps frames differ little).
6. The pipeline hooks: ``prepare_audio_embeddings`` (a stub encoder with a fixed last_hidden_state) and
   ``prepare_kps_feature``, L = 20 with CFG, against the fp64 composition under the section 3 thresholds.

With every attention branch zeroed, the latents never see x, so the feed-forward cases check the ff branch on the
five learned latent rows whatever the input; the attention cases carry the input dependence.

Thresholds: FLOOR = 1e-2 and CEIL = 2e-2, below half the smallest module-level fault (7.5e-2).  Measured on an H100
80GB HBM3 at its 700 W power limit (e_eager of the oracle in bf16 on the same GPU):
    worst bound ratio per call kind, over every call of the section 1 forwards and the im2col cases:
        conv_in 0.985, im2col 0.996, gemm 0.950, geglu 0.827, layernorm 0.993, attention 0.50 -- the output rounding
    guider (v-kps, noise, black; 512^2 b 1 / 2 t 16, 768^2 t 8): e_eager 2.36e-3 - 3.09e-3, e_prod 2.20e-3 - 2.61e-3
        (at most 0.26 of the threshold)
    projection branches (attn / ff of each layer at gain 1, share 1.34 - 1.38): e_eager 3.1e-3 - 4.8e-3, e_prod
        2.6e-3 - 3.9e-3 (at most 0.39);  path alone 2.29e-3 / 2.29e-3;  whole module at L = 300: e_eager 9.75e-3,
        e_prod 7.98e-3 (0.55, the largest)
    pipeline hooks at L = 20: prepare_audio_embeddings e_prod 8.39e-3 (e_eager 1.02e-2, 0.55 of the threshold),
        prepare_kps_feature 2.18e-3 (0.22)
FLOOR keeps a case whose eager run is unusually accurate from a threshold tighter than storing its output in bf16.
The GPU cases of this file take about 25 s.
"""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import vx_oracle as O
from test_attention_bounds_gpu import attention_ref64
from test_attention_bounds_gpu import bound_check as attn_bound_check
from test_gemm_bounds_gpu import (_SENTINEL, _chunks, _conv_in_ref64, _sentinel_buf, bound_check, geglu_ref64,
                                  linear_bound, linear_ref64)
from test_norm_bounds_gpu import _act_terms, _silu64, layernorm_ref64

BF16, F64 = torch.bfloat16, torch.float64
KPS, AP = O.KPS_CFG, O.AUDIO_PROJ_CFG
FLOOR, CEIL = 1e-2, 2e-2
MIN_SHARE = 0.5
GLOBAL = {"conv_in": 5e-3, "im2col": 5e-3, "gemm": 5e-3, "geglu": 5e-3, "layernorm": 5e-3, "attention": 4e-3}
_WORST = {}                    # call kind -> (worst bound ratio, case)
RESULTS = []                   # (case, e_prod, e_eager, share, threshold)


# ------------------------------------------------------------------------------------------------------------ helpers
def _seed(*xs):
    s = 0
    for v in xs:
        s = (s * 1000003 + sum(map(ord, str(v)))) % (1 << 31)
    return s


def _gen(*xs):
    return torch.Generator().manual_seed(_seed(*xs))


def _norm(t):
    return float(t.double().norm())


def _measure(out, ref, B):
    return _norm(out.double() - ref) / max(_norm(B), 1e-30)


def threshold(e_eager):
    return min(max(1.5 * e_eager, FLOOR), CEIL)


def im2col_ref(Y, stride, pad_lo=1):
    """The kernel's gather of NHWC Y (n, H, W, C) -> [n Ho Wo, 9 C], (tap, channel) order, zero padding, in Y's dtype."""
    n, H, W, C = Y.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    p = F.pad(Y, (0, 0, pad_lo, 2, pad_lo, 2))
    taps = [p[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
            for ky in range(3) for kx in range(3)]
    return torch.cat(taps, -1).reshape(n * Ho * Wo, 9 * C)


def im2col_sources(col, n, H, W, C, stride, pad_lo=1):
    """The per-pixel values (n, H, W, C) a gather wrote, read back from its taps (every pixel is some tap's source)."""
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    cv = col.view(n, Ho, Wo, 9, C)
    Y = torch.zeros((n, H + 4, W + 4, C), dtype=col.dtype, device=col.device)
    for t in range(9):
        y0, x0 = 2 + t // 3 - pad_lo, 2 + t % 3 - pad_lo
        Y[:, y0:y0 + stride * (Ho - 1) + 1:stride, x0:x0 + stride * (Wo - 1) + 1:stride] = cv[:, :, :, t]
    return Y[:, 2:2 + H, 2:2 + W]


def silu_ref64(x):
    """(ref, bound without the output rounding) of the gather's SiLU x / (1 + __expf(-x)) (module docstring)."""
    xd = x.double()
    return _silu64(xd), _act_terms(xd, torch.zeros_like(xd))[1]


def check_im2col(x, col, n, H, W, stride, silu, pad_lo=1):
    """'' or a failure: col must be the bit-exact gather of per-pixel values that equal x (no SiLU) or are within the
    SiLU bound of x.  Frame by frame, so that the fp64 temporaries stay small."""
    C = x.shape[1]
    HW = H * W
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    rows = Ho * Wo
    worst, where, err2, ref2 = 0.0, "", 0.0, 0.0
    for f in range(n):
        c = col[f * rows:(f + 1) * rows]
        Y = im2col_sources(c, 1, H, W, C, stride, pad_lo)
        if not torch.equal(c.view(torch.int16), im2col_ref(Y, stride, pad_lo).view(torch.int16)):
            bad = (c.view(torch.int16) != im2col_ref(Y, stride, pad_lo).view(torch.int16)).nonzero()[0].tolist()
            return f"gather not bit-exact in frame {f}, first at (row, column) {bad}"
        xs = x[f * HW:(f + 1) * HW].view(1, H, W, C)
        if not silu:
            if not torch.equal(Y.view(torch.int16), xs.view(torch.int16)):
                return f"gathered values differ from x in frame {f}"
            continue
        ref, bnd = silu_ref64(xs.reshape(HW, C))
        w, _, wh = bound_check(Y.reshape(HW, C), ref, bnd)
        if w > worst:
            worst, where = w, f"frame {f} {wh}"
        err2 += _norm(Y.reshape(HW, C).double() - ref) ** 2
        ref2 += _norm(ref) ** 2
    if silu:
        return _verdict("im2col", f"n {n} {H}x{W} C {C} s{stride}", worst, where, math.sqrt(err2 / max(ref2, 1e-300)))
    return ""


def _verdict(kind, case, worst, where, rel):
    print(f"  {kind:9s} {case}: worst ratio {worst:.3f}, rel {rel:.2e}")
    if worst > _WORST.get(kind, (-1.0, ""))[0]:
        _WORST[kind] = (worst, case)
    bad = []
    if not worst <= 1:
        bad.append(f"bound exceeded, {where}")
    if not rel < GLOBAL[kind]:
        bad.append(f"global rel {rel:.3e}")
    return f"{kind} {case}: " + "; ".join(bad) if bad else ""


def _judge_rows(kind, case, out, rows, ref_fn, residual=None, step=None):
    """Judge out [rows, N] chunk by chunk: ref_fn(r0, r1) -> (ref, bound without output rounding)."""
    worst, where, e2, r2, d2 = 0.0, "", 0.0, 0.0, 0.0
    step = step or rows
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        ref, bnd = ref_fn(r0, r1)
        o = out[r0:r1]
        w, _, wh = bound_check(o, ref, bnd)
        if w > worst:
            worst, where = w, f"rows {r0}+ {wh}"
        e2 += _norm(o.double() - ref) ** 2
        r2 += _norm(ref) ** 2
        if residual is not None:
            d2 += _norm(ref - residual[r0:r1].double()) ** 2
    return _verdict(kind, case, worst, where, math.sqrt(e2 / max(r2, d2, 1e-300)))


def _geglu_unpack(ops, wp, bp):
    """Invert pack_geglu: the [value rows | gate rows] weights and bias the packed ones came from."""
    N = wp.shape[0]
    idx = ops.pack_geglu(torch.arange(N, device=wp.device)[:, None], None)[0][:, 0]
    w, b = torch.empty_like(wp), torch.empty_like(bp)
    w[idx], b[idx] = wp, bp
    return w, b


class _Recorder:
    """Stands in for ``ops`` inside modules/prologue.py: forwards each call to the real ops, then judges its output
    against the fp64 reference of the operands it read.  Failures collect in ``fails``; with ``widths`` (the guider's
    true output widths per layer) the padded columns must be 0, and with ``uniform`` (all-black frames) every pixel
    untouched by the zero padding must hold the same bits at every layer; ``judge=False`` skips the fp64 references."""

    def __init__(self, real, case, widths=None, uniform=False, judge=True):
        self.real, self.case, self.widths, self.uniform, self.judge = real, case, widths, uniform, judge
        self.fails, self.counts = [], {}
        self._layer, self._geom, self._taint = 0, None, None

    def __getattr__(self, name):
        return getattr(self.real, name)

    def _done(self, kind, msg):
        self.counts[kind] = self.counts.get(kind, 0) + 1
        if msg and self.judge:
            self.fails.append(f"{self.case}: {msg}")

    def _guider_checks(self, out, n, h, w):
        if self.widths is not None:
            real = self.widths[self._layer]
            if real < out.shape[1] and out[:, real:].abs().amax() != 0:
                self.fails.append(f"{self.case}: layer {self._layer} padded columns {real}.. not zero")
        if self.uniform:
            bits = out.view(torch.int16).view(n, h, w, -1)
            keep = ~self._taint.view(1, h, w).expand(n, h, w)
            inner = bits[keep]
            if inner.shape[0] and not bool((inner == inner[:1]).all()):
                self.fails.append(f"{self.case}: layer {self._layer} interior pixels of black frames differ")
        self._layer += 1

    def conv_in(self, x, w, bias, Cout, **kw):
        out = self.real.conv_in(x, w, bias, Cout, **kw)
        n, cin, H, W = x.shape
        assert not kw
        step = max(1, (1 << 27) // (H * W * Cout * 8))
        case = f"{self.case} n {n} {H}x{W} 4->{Cout}"
        wt = w.t().reshape(Cout, cin, 3, 3)
        self._done("conv_in", self.judge and _judge_rows("conv_in", case, out, n * H * W,
                                          lambda r0, r1: _conv_in_ref64(x[r0 // (H * W):r1 // (H * W)], wt, bias),
                                          step=step * H * W))
        self._layer, self._geom = 0, (n, H, W)
        self._taint = torch.zeros((H, W), dtype=torch.bool, device=x.device)
        self._guider_checks(out, n, H, W)
        return out

    def im2col3x3(self, x, n, h, w, stride=1, silu=False, **kw):
        col = self.real.im2col3x3(x, n, h, w, stride=stride, silu=silu, **kw)
        pad_lo = kw.get("pad_lo", 1)
        self._done("im2col", self.judge and check_im2col(x, col, n, h, w, stride, silu, pad_lo))
        if self._taint is not None:
            t = F.pad(self._taint.float()[None, None], (1, 1, 1, 1), value=1.0)
            self._taint = F.max_pool2d(t, 3, stride)[0, 0] > 0
        self._geom = (n, (h - 1) // stride + 1, (w - 1) // stride + 1)
        return col

    def gemm(self, a, w, bias=None, *, residual=None, geglu=False, **kw):
        out = self.real.gemm(a, w, bias, residual=residual, geglu=geglu, **kw)
        assert not kw, kw
        M, K = a.shape
        case = f"{self.case} M {M} K {K} N {w.shape[0]}"
        if not self.judge:
            self._done("geglu" if geglu else "gemm", "")
        elif geglu:
            wu, bu = _geglu_unpack(self.real, w, bias)
            step = _chunks(M, K, 8 * w.shape[0])[0][1]
            self._done("geglu", _judge_rows("geglu", case, out, M, lambda r0, r1: geglu_ref64(a[r0:r1], wu, bu),
                                            step=step))
        else:
            def ref(r0, r1):
                r, ra, p = linear_ref64(a[r0:r1], w, bias, residual=None if residual is None else residual[r0:r1])
                return r, linear_bound(r, ra, p, K)
            self._done("gemm", _judge_rows("gemm", case, out, M, ref, residual, step=_chunks(M, K, w.shape[0])[0][1]))
        if self._geom is not None:
            self._guider_checks(out, *self._geom)
        return out

    def layernorm(self, x, gamma, beta, eps=1e-5, **kw):
        out = self.real.layernorm(x, gamma, beta, eps, **kw)
        assert not kw
        self._done("layernorm", self.judge and _judge_rows("layernorm", f"{self.case} rows {x.shape[0]} C {x.shape[1]}", out,
                                            x.shape[0], lambda r0, r1: layernorm_ref64(x[r0:r1], gamma, beta, eps)))
        return out

    def flash_attention(self, q, k, v, heads, Nq, Nk, **kw):
        out = self.real.flash_attention(q, k, v, heads, Nq, Nk, **kw)
        assert not kw
        if not self.judge:
            self._done("attention", "")
            return out
        ref, ref_abs = attention_ref64(q, k, v, heads, Nq, Nk)
        worst, rel, where = attn_bound_check(out, ref, ref_abs, Nk, Nq, heads)
        self._done("attention", _verdict("attention", f"{self.case} B {q.shape[0] // Nq} {Nq}x{Nk} x{heads}", worst,
                                         where, rel))
        return out


# --------------------------------------------------------------------------------------------------------- input data
def vkps_frames(b, t, H, W, seed):
    """(b, 3, t, H, W) in [0, 1] after the reference's draw_v_kps_image: a black canvas, two sticks of half-width 4 at
    intensity 0.6 joining three keypoints, and a radius-4 dot on each keypoint in R, G and B.  The keypoints move from
    frame to frame, so a permuted frame or chunk shows."""
    g = _gen("vkps", b, t, H, W, seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    img = torch.zeros(b, 3, t, H, W)
    hw = torch.tensor([H, W], dtype=torch.float32)
    for s in range(b):
        base = 0.25 + 0.5 * torch.rand(3, 2, generator=g)
        vel = 0.03 * (torch.rand(3, 2, generator=g) - 0.5)
        for f in range(t):
            p = (base + vel * f) * hw
            for (i, j), colour in (((0, 1), (0.6, 0.6, 0.0)), ((1, 2), (0.0, 0.6, 0.6))):
                a, d = p[i], p[j] - p[i]
                u = (((yy - a[0]) * d[0] + (xx - a[1]) * d[1]) / float((d * d).sum().clamp_min(1e-6))).clamp(0, 1)
                m = (yy - a[0] - u * d[0]) ** 2 + (xx - a[1] - u * d[1]) ** 2 <= 16
                for ch in range(3):
                    img[s, ch, f][m] = colour[ch]
            for k in range(3):
                img[s, k, f][(yy - p[k, 0]) ** 2 + (xx - p[k, 1]) ** 2 <= 16] = 1.0
    return img


def kps_inputs(fam, b, t, H, W, seed=0):
    if fam == "v-kps":
        return vkps_frames(b, t, H, W, seed)
    if fam == "noise":
        return torch.rand(b, 3, t, H, W, generator=_gen("noise", b, t, H, W, seed))
    return torch.zeros(b, 3, t, H, W)


def audio_inputs(fam, L, seed=0):
    """(L, 10, 768) bf16 windows.  wav2vec: states (1, T, 768) with per-channel scales through audio_frame_windows;
    jumpy: every window its own scale (4^(l mod 3)) and offset, so a frame that reads its neighbour's window shows."""
    g = _gen("audio", fam, L, seed)
    if fam == "wav2vec":
        T = 2 * L + 7
        states = torch.randn(1, T, 768, generator=g) * (0.2 + 2 * torch.rand(768, generator=g))
        return O.audio_frame_windows(states.to(BF16), L)
    s = 4.0 ** (torch.arange(L) % 3).float()[:, None, None]
    return (torch.randn(L, 10, 768, generator=g) * s + torch.randn(L, 1, 768, generator=g)).to(BF16)


# ------------------------------------------------------------------------------------------------------ state dicts
def _guider_sd(seed=11):
    return {k: v.to(BF16).double() for k, v in O.synth_state_dict(O.kps_guider_param_shapes(KPS), seed).items()}


def _proj_sd(seed=12):
    """Synthetic weights (bf16 values, held in fp64) with pos_emb and the LayerNorm parameters redrawn (docstring)."""
    sd = O.synth_state_dict(O.audio_projection_param_shapes(AP), seed)
    g = _gen("proj-sd", seed)
    for k in sorted(sd):
        if k == "pos_emb.weight":
            sd[k] = 0.5 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith(("norm1.weight", "norm2.weight", ".1.0.weight", "norm_out.weight")):
            sd[k] = 1 + 0.25 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith(("norm1.bias", "norm2.bias", ".1.0.bias", "norm_out.bias")):
            sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
    return {k: v.to(BF16).double() for k, v in sd.items()}


def branch_key(i, br):
    return f"layers.{i}.0.to_out.weight" if br == "attn" else f"layers.{i}.1.3.weight"


def isolate(sd, keep=None, gain=1.0, drop_keep=False):
    """Zero every branch's output weight but ``keep`` = (layer, branch), scale that one by ``gain`` (or zero it too)."""
    out = dict(sd)
    for i in range(AP["depth"]):
        for br in ("attn", "ff"):
            s = 0.0 if ((i, br) != keep or drop_keep) else gain
            if s != 1.0:
                out[branch_key(i, br)] = sd[branch_key(i, br)] * s
    return out


# ------------------------------------------------------------------------------ fault-injectable fp64 models (CPU)
GUIDER_FAULTS = ("no_silu_after_conv_in", "silu_after_conv_out", "stride2_on_same_width_conv", "stride2_pad_0101",
                 "im2col_k_channel_major", "frame_across_chunk", "conv_out_bias_dropped")
PROJ_FAULTS = ("pos_emb_shifted", "scale_1_over_hd", "kv_without_latents", "kv_halves_swapped", "norm1_norm2_swapped",
               "window_of_next_frame", "norm_out_dropped")


def guider64(sd, x, fault=None, frames_per_chunk=8):
    """O.kps_guider_forward with an injectable fault (x (b, 3, t, H, W), any float dtype; sd in the same dtype)."""
    b, c, t, H, W = x.shape
    h = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, H, W)
    if fault == "frame_across_chunk":
        h = h.clone()
        h[frames_per_chunk - 1] = h[frames_per_chunk]

    def conv(name, v, stride):
        w, bias, pad = sd[name + ".weight"], sd[name + ".bias"], 1
        if fault == "stride2_pad_0101" and stride == 2:
            v, pad = F.pad(v, (0, 1, 0, 1)), 0
        if fault == "im2col_k_channel_major" and name != "conv_in":
            co, ci = w.shape[:2]
            w = w.reshape(co, 9 * ci).reshape(co, 3, 3, ci).permute(0, 3, 1, 2)
        if fault == "conv_out_bias_dropped" and name == "conv_out":
            bias = None
        return F.conv2d(v, w, bias, stride=stride, padding=pad)

    h = conv("conv_in", h, 1)
    if fault != "no_silu_after_conv_in":
        h = F.silu(h)
    for i in range(2 * (len(KPS["block_out_channels"]) - 1)):
        stride = (2 - (i & 1)) if fault == "stride2_on_same_width_conv" else 1 + (i & 1)
        h = F.silu(conv(f"blocks.{i}", h, stride))
    h = conv("conv_out", h, 1)
    if fault == "silu_after_conv_out":
        h = F.silu(h)
    return h.view(b, t, *h.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()


def proj64(sd, x, fault=None, gelu="none"):
    """O.audio_projection_forward with an injectable fault; gelu 'tanh' swaps in the tanh-form GELU."""
    heads, hd = AP["heads"], AP["dim_head"]
    L, n, _ = x.shape
    if fault == "window_of_next_frame":
        x = torch.cat([x[1:], x[-1:]])
    pe = sd["pos_emb.weight"][:n]
    if fault == "pos_emb_shifted":
        pe = sd["pos_emb.weight"][torch.arange(1, n + 1) % sd["pos_emb.weight"].shape[0]]
    x = F.linear(x + pe, sd["proj_in.weight"], sd["proj_in.bias"])
    lat = sd["latents"].repeat(L, 1, 1)
    ln_ = lambda p, v: F.layer_norm(v, (v.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)
    split = lambda t: t.view(t.shape[0], t.shape[1], heads, hd).transpose(1, 2)
    for i in range(AP["depth"]):
        a, f = f"layers.{i}.0", f"layers.{i}.1"
        n1, n2 = ("norm2", "norm1") if fault == "norm1_norm2_swapped" else ("norm1", "norm2")
        xn, ln = ln_(f"{a}.{n1}", x), ln_(f"{a}.{n2}", lat)
        q = split(F.linear(ln, sd[a + ".to_q.weight"]))
        kv_in = xn if fault == "kv_without_latents" else torch.cat([xn, ln], 1)
        k, v = F.linear(kv_in, sd[a + ".to_kv.weight"]).chunk(2, -1)
        if fault == "kv_halves_swapped":
            k, v = v, k
        s = 1 / hd if fault == "scale_1_over_hd" else 1 / math.sqrt(hd)
        o = torch.softmax(q @ split(k).transpose(-1, -2) * s, -1) @ split(v)
        lat = F.linear(o.transpose(1, 2).reshape(L, -1, heads * hd), sd[a + ".to_out.weight"]) + lat
        hh = F.linear(ln_(f + ".0", lat), sd[f + ".1.weight"])
        lat = F.linear(F.gelu(hh, approximate="tanh" if gelu == "tanh" else "none"), sd[f + ".3.weight"]) + lat
    out = F.linear(lat, sd["proj_out.weight"], sd["proj_out.bias"])
    return out if fault == "norm_out_dropped" else ln_("norm_out", out)


# -------------------------------------------------------------------------------------------------------- the cases
def proj_cases(sd, x, run, with_whole=True):
    """Section 3 cases of the perceiver: [(name, sd_case, B-zero sd or None, share-gain)] evaluated by ``run(sd, x)``
    (an fp64 forward) -> list of dicts with name, sd, ref, B, share."""
    cases = []
    for i in range(AP["depth"]):
        for br in ("attn", "ff"):
            gain = 1.0
            while True:
                sdc = isolate(sd, (i, br), gain)
                ref = run(sdc, x)
                B = ref - run(isolate(sd, (i, br), drop_keep=True), x)
                share = _norm(B) / max(_norm(ref), 1e-30)
                if share >= MIN_SHARE or gain >= 64:
                    break
                gain *= 2
            cases.append(dict(name=f"layer {i} {br} x{gain:g}", sd=sdc, ref=ref, B=B, share=share))
    sdp = isolate(sd)
    ref = run(sdp, x)
    cases.append(dict(name="path alone", sd=sdp, ref=ref, B=ref, share=1.0))
    if with_whole:
        ref = run(sd, x)
        cases.append(dict(name="whole", sd=sd, ref=ref, B=ref, share=1.0))
    return cases


def _record(name, e_prod, e_eager, share, finite=True):
    thr = threshold(e_eager)
    RESULTS.append((name, e_prod, e_eager, share, thr))
    print(f"{name:52s} e_prod {e_prod:.3e}  e_eager {e_eager:.3e}  share {share:.2f}  thr {thr:.2e}  "
          f"({e_prod / thr:.2f} of it)")
    if not finite:
        return f"{name}: NaN / Inf in the output"
    if not e_prod <= thr:
        return f"{name}: e_prod {e_prod:.3e} > threshold {thr:.3e} (e_eager {e_eager:.3e})"
    return ""


# ------------------------------------------------------------------------------------------------------ CPU self-tests
def test_fp64_models_equal_the_oracle():
    sd = _guider_sd()
    x = vkps_frames(1, 3, 32, 32, 0).double()
    torch.testing.assert_close(guider64(sd, x), O.kps_guider_forward(sd, KPS, x), rtol=1e-12, atol=1e-12)
    sdp = _proj_sd()
    xa = audio_inputs("wav2vec", 4).double()
    # the oracle takes its softmax in fp32 (as the reference does): agreement to fp32 accuracy
    torch.testing.assert_close(proj64(sdp, xa), O.audio_projection_forward(sdp, AP, xa), rtol=1e-5, atol=2e-6)


def test_im2col_reference_matches_unfold_and_round_trips():
    g = _gen("im2col-cpu")
    for (n, H, W, C, stride, pad_lo) in [(2, 7, 9, 8, 1, 1), (2, 7, 9, 8, 2, 1), (1, 8, 6, 16, 2, 0)]:
        Y = torch.randn(n, H, W, C, generator=g).double()
        col = im2col_ref(Y, stride, pad_lo)
        x = Y.permute(0, 3, 1, 2)
        if pad_lo == 0:
            x = F.pad(x, (0, 1, 0, 1))
        u = F.unfold(x, 3, padding=pad_lo, stride=stride)
        ref = u.view(n, C, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * C)
        assert torch.equal(col, ref)
        assert torch.equal(im2col_sources(col, n, H, W, C, stride, pad_lo), Y)


def test_silu_bound_self_test():
    """The kernel's SiLU form (fp32 x / (1 + exp(-x)), bf16 out) stays inside the bound over the whole bf16 range that
    matters; a SiLU rounded twice does not."""
    x = torch.linspace(-100, 30, 200001).to(BF16).unique()
    ref, bnd = silu_ref64(x)
    xf = x.float()
    good = (xf / (1 + torch.exp(-xf))).to(BF16)
    assert bound_check(good, ref, bnd)[0] <= 1
    twice = (xf * torch.sigmoid(xf).to(BF16).float()).to(BF16)
    assert bound_check(twice, ref, bnd)[0] > 1.5
    tanh = (0.5 * xf * (1 + torch.tanh(0.5 * xf)).to(BF16).float()).to(BF16)
    assert bound_check(tanh, ref, bnd)[0] > 1.5


def test_recorder_judges_emulated_forward(monkeypatch):
    """The recorder's checks on the CPU emulation of the kernels (tests/test_host_cpu.py): every call kind is judged and
    passes, the padded columns are zero and black frames give uniform interiors."""
    from test_host_cpu import _EmuOps
    from vexpress_b200 import _ffi
    from vexpress_b200.modules import prologue
    monkeypatch.setattr(_ffi, "require_sm90", lambda: None)
    emu = _EmuOps()
    m = prologue.VKpsGuider(320, block_out_channels=(16, 32, 96, 256))
    m.load_state_dict({k: v.float() for k, v in _guider_sd().items()})
    m = m.to(BF16)
    for fam in ("v-kps", "black"):
        rec = _Recorder(emu, f"cpu {fam}", widths=_guider_widths(), uniform=fam == "black")
        monkeypatch.setattr(prologue, "ops", rec)
        m(kps_inputs(fam, 1, 3, 32, 32), frames_per_chunk=2)
        assert not rec.fails, "\n".join(rec.fails)
        assert rec.counts == {"conv_in": 2, "im2col": 14, "gemm": 14}, rec.counts
    p = prologue.AudioProjection(**AP)
    p.load_state_dict({k: v.float() for k, v in _proj_sd().items()})
    p = p.to(BF16)
    rec = _Recorder(emu, "cpu proj")
    monkeypatch.setattr(prologue, "ops", rec)
    p(audio_inputs("wav2vec", 3))
    assert not rec.fails, "\n".join(rec.fails)
    assert rec.counts == {"gemm": 18, "layernorm": 13, "attention": 4, "geglu": 4}, rec.counts


def _guider_widths():
    boc = KPS["block_out_channels"]
    return [boc[0], boc[0], boc[1], boc[1], boc[2], boc[2], boc[3], KPS["conditioning_embedding_channels"]]


def _fault_cases_guider():
    sd = _guider_sd()
    out = []
    for fam in ("v-kps", "noise"):
        x = kps_inputs(fam, 1, 4, 64, 64, seed=1).to(BF16)
        ref = guider64(sd, x.double(), frames_per_chunk=2)
        eager = O.kps_guider_forward({k: v.to(BF16) for k, v in sd.items()}, KPS, x)
        out.append(dict(name=f"guider {fam}", sd=sd, x=x, ref=ref, B=ref, e_eager=_measure(eager, ref, ref)))
    return out


def _fault_cases_proj():
    sd = _proj_sd()
    out = []
    for fam in ("wav2vec", "jumpy"):
        x = audio_inputs(fam, 6, seed=1)
        for c in proj_cases(sd, x.double(), lambda s, v: O.audio_projection_forward(s, AP, v)):
            eager = O.audio_projection_forward({k: v.to(BF16) for k, v in c["sd"].items()}, AP, x)
            c.update(name=f"{fam} {c['name']}", x=x, e_eager=_measure(eager, c["ref"], c["B"]))
            out.append(c)
    return out


def test_fault_catalogue():
    """Each composition fault moves the measure of at least one case by 2x its threshold; the oracle's own bf16 run
    passes every case (the CPU self-test of the check)."""
    table = []
    for cases, faults, model in ((_fault_cases_guider(), GUIDER_FAULTS, lambda c, f: guider64(c["sd"], c["x"].double(), f, 2)),
                                 (_fault_cases_proj(), PROJ_FAULTS, lambda c, f: proj64(c["sd"], c["x"].double(), f))):
        for c in cases:
            assert c["share"] >= MIN_SHARE if "share" in c else True, (c["name"], c["share"])
            assert c["e_eager"] <= threshold(c["e_eager"]), c["name"]
        for fault in faults:
            best = max(((_measure(model(c, fault), c["ref"], c["B"]), threshold(c["e_eager"]), c["name"]) for c in cases),
                       key=lambda t: t[0] / t[1])
            table.append((fault, *best))
    # tanh-GELU: judged where the recorder sees it, the GEGLU call of layer 0's feed-forward
    sd = _proj_sd()
    x = audio_inputs("wav2vec", 6, seed=1).double()
    lat = sd["latents"].repeat(x.shape[0], 1, 1)
    h = F.layer_norm(lat, (768,), sd["layers.0.1.0.weight"], sd["layers.0.1.0.bias"], 1e-5).to(BF16).reshape(-1, 768)
    w1 = sd["layers.0.1.1.weight"]
    wv = torch.cat([torch.zeros_like(w1), w1], 0)
    bv = torch.cat([torch.ones(w1.shape[0]), torch.zeros(w1.shape[0])]).double()
    ref, bnd = geglu_ref64(h, wv, bv)
    pre = h.double() @ w1.t()
    tanh_out = F.gelu(pre.float(), approximate="tanh").to(BF16)
    ratio = bound_check(tanh_out, ref, bnd)[0]
    erf_ratio = bound_check(F.gelu(pre.float()).to(BF16), ref, bnd)[0]
    print(f"{'gelu_tanh (GEGLU call bound)':34s} worst ratio {ratio:.2f} (erf form {erf_ratio:.2f})")
    for fault, e, thr, name in table:
        print(f"{fault:34s} {e:.3e} / {thr:.2e} = {e / thr:6.2f}  ({name})")
    assert erf_ratio <= 1 and ratio >= 2
    missed = [f"{fault}: {e:.3e} < 2 x {thr:.2e}" for fault, e, thr, _ in table if not e >= 2 * thr]
    assert not missed, "\n".join(missed)


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for kind, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {kind:10s} {worst:.3f}  ({case})")
    for name, e, ee, share, thr in RESULTS:
        print(f"{name:52s} e_prod {e:.3e} e_eager {ee:.3e} share {share:.2f} thr {thr:.2e} ({e / thr:.2f})")


@pytest.fixture(scope="module")
def guider():
    from vexpress_b200.modules.prologue import VKpsGuider
    sd = _guider_sd()
    m = VKpsGuider(KPS["conditioning_embedding_channels"], block_out_channels=KPS["block_out_channels"])
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    return m.to(device="cuda", dtype=BF16), {k: v.cuda() for k, v in sd.items()}


@pytest.fixture(scope="module")
def projection():
    from vexpress_b200.modules.prologue import AudioProjection
    sd = _proj_sd()
    p = AudioProjection(**AP)
    p.load_state_dict({k: v.float() for k, v in sd.items()})
    return p.to(device="cuda", dtype=BF16), {k: v.cuda() for k, v in sd.items()}


def _load(module, sd):
    module.load_state_dict({k: v.float() for k, v in sd.items()})
    return module.to(device="cuda", dtype=BF16)


# ---- 1. every kernel call of a real forward
@pytest.mark.gpu
@pytest.mark.parametrize("size,frames", [(512, 8), (512, 5), (768, 8), (768, 5)])
def test_guider_every_call_within_bound(ops, guider, monkeypatch, size, frames):
    from vexpress_b200.modules import prologue
    m, _ = guider
    rec = _Recorder(ops, f"guider {size}^2 bt {frames}", widths=_guider_widths())
    monkeypatch.setattr(prologue, "ops", rec)
    with torch.no_grad():
        y = m(kps_inputs("v-kps", 1, frames, size, size, seed=size).cuda())
    torch.cuda.synchronize()
    assert rec.counts == {"conv_in": 1, "im2col": 7, "gemm": 7}, rec.counts
    assert bool(torch.isfinite(y.float()).all())
    assert not rec.fails, "\n".join(rec.fails)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 7, 300, 1000])
def test_projection_every_call_within_bound(ops, projection, monkeypatch, L):
    from vexpress_b200.modules import prologue
    p, _ = projection
    rec = _Recorder(ops, f"projection L {L}")
    monkeypatch.setattr(prologue, "ops", rec)
    with torch.no_grad():
        p(audio_inputs("wav2vec" if L % 2 else "jumpy", L).cuda())
    torch.cuda.synchronize()
    assert rec.counts == {"gemm": 18, "layernorm": 13, "attention": 4, "geglu": 4}, rec.counts
    assert not rec.fails, "\n".join(rec.fails)


# ---- 2. im2col3x3 on its own
@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,stride,pad_lo", [(2, 16, 16, 32, 1, 1), (3, 33, 17, 96, 1, 1), (2, 16, 24, 32, 2, 1),
                                                    (3, 33, 17, 96, 2, 1), (2, 15, 9, 32, 2, 1), (2, 16, 24, 96, 2, 0),
                                                    (1, 64, 64, 32, 2, 0)])
@pytest.mark.parametrize("silu", [False, True])
def test_im2col3x3_gather_and_silu(ops, NB, H, W, C, stride, pad_lo, silu):
    g = torch.Generator(device="cuda").manual_seed(_seed(NB, H, W, C, stride, pad_lo))
    HW = H * W
    xb = torch.full(((NB + 2) * HW, C), float("nan"), device="cuda", dtype=BF16)
    x = xb[HW:(NB + 1) * HW]
    x.copy_(torch.randn(NB * HW, C, device="cuda", generator=g) * 6)    # down to the exp overflow: -30 .. 30
    x[:8] = torch.tensor([-100.0, -89.0, -88.0, -20.0, -0.0, 0.0, 1e-30, 80.0], device="cuda").to(BF16)[:, None]
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    rows = NB * Ho * Wo
    buf = _sentinel_buf((rows + 8, 9 * C))
    out = buf[3:3 + rows]
    ret = ops.im2col3x3(x, NB, H, W, stride=stride, silu=silu, out=out, pad_lo=pad_lo)
    torch.cuda.synchronize()
    assert ret.data_ptr() == out.data_ptr()
    border = torch.cat([buf[:3], buf[3 + rows:]]).view(torch.int16)
    assert bool((border == _SENTINEL).all()), "im2col3x3 wrote outside its output"
    msg = check_im2col(x, out, NB, H, W, stride, silu, pad_lo)
    assert not msg, msg


@pytest.mark.gpu
def test_im2col3x3_rejects_strided_views(ops):
    x = torch.zeros(4 * 4, 64, device="cuda", dtype=BF16)
    with pytest.raises(ValueError):
        ops.im2col3x3(x[:, :32], 1, 4, 4)
    out = torch.zeros(16, 9 * 64, device="cuda", dtype=BF16)
    with pytest.raises(ValueError):
        ops.im2col3x3(x[:, :32].contiguous(), 1, 4, 4, out=out[:, :9 * 32])


# ---- 3. modules against fp64 with the eager yardstick
@pytest.mark.gpu
@pytest.mark.parametrize("fam", ["wav2vec", "jumpy"])
def test_projection_branches_against_fp64(projection, fam):
    p, sd = projection
    L = 300 if fam == "wav2vec" else 64
    x = audio_inputs(fam, L, seed=3).cuda()
    fails = []
    for c in proj_cases(sd, x.double(), lambda s, v: O.audio_projection_forward(s, AP, v), with_whole=(fam == "wav2vec")):
        assert c["share"] >= MIN_SHARE, (c["name"], c["share"])
        with torch.no_grad():
            eager = O.audio_projection_forward({k: v.to(BF16) for k, v in c["sd"].items()}, AP, x)
            out = _load(p, c["sd"])(x)
        fails.append(_record(f"projection {fam} L {L} {c['name']}", _measure(out, c["ref"], c["B"]),
                             _measure(eager, c["ref"], c["B"]), c["share"], bool(torch.isfinite(out.float()).all())))
    _load(p, sd)
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


def _guider_ref(sd, x, dtype):
    """The oracle guider on the GPU in ``dtype``, one frame at a time (b t frames at 768^2 in fp64 are several GB)."""
    b, c, t, H, W = x.shape
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    frames = [O.kps_guider_forward(sdd, KPS, x[:, :, j:j + 1].to(dtype)) for j in range(t)]
    return torch.cat(frames, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("size,b,t", [(512, 1, 16), (512, 2, 16), (768, 1, 8)])
@pytest.mark.parametrize("fam", ["v-kps", "noise", "black"])
def test_guider_against_fp64(ops, guider, monkeypatch, size, b, t, fam):
    from vexpress_b200.modules import prologue
    m, sd = guider
    x = kps_inputs(fam, b, t, size, size, seed=size + b).to(BF16).cuda()
    rec = None
    if fam == "black":
        rec = _Recorder(ops, f"guider black {size}^2", uniform=True, judge=False)
        monkeypatch.setattr(prologue, "ops", rec)
    with torch.no_grad():
        out = m(x)
        ref = _guider_ref(sd, x, F64)
        eager = _guider_ref(sd, x, BF16)
    msg = _record(f"guider {fam} {size}^2 b {b} t {t}", _measure(out, ref, ref), _measure(eager, ref, ref), 1.0,
                  bool(torch.isfinite(out.float()).all()))
    assert not msg, msg
    if rec is not None:
        assert not rec.fails, "\n".join(rec.fails)


# ---- 4. batching and chunking invariants, bit-exact
def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.mark.gpu
def test_guider_chunking_is_bit_exact(guider):
    m, _ = guider
    x = kps_inputs("v-kps", 2, 8, 256, 256, seed=5).cuda()
    with torch.no_grad():
        base = m(x[:1])
        for fpc in (1, 3, 8):
            assert _bits_equal(m(x[:1], frames_per_chunk=fpc), base), f"frames_per_chunk {fpc}"
        rev = m(x[:1].flip(2))
        assert _bits_equal(rev.flip(2), base), "frame position within the chunk"
        both = m(x, frames_per_chunk=3)
        assert _bits_equal(both[:1], base), "b = 2, sample 0"
        assert _bits_equal(both[1:], m(x[1:])), "b = 2, sample 1"


class _Dev:
    device, dtype = torch.device("cuda"), BF16


def _pipeline(guider=None, projection=None, states=None):
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    enc = None
    if states is not None:
        enc = lambda wave: types.SimpleNamespace(last_hidden_state=states)
    return VExpressPipeline(vae=None, reference_net=None, denoising_unet=_Dev(), v_kps_guider=guider,
                            audio_processor=None, audio_encoder=enc, audio_projection=projection, scheduler=None)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 16, 17, 20, 33])
@pytest.mark.parametrize("cfg", [True, False])
def test_prepare_kps_feature_is_per_frame_guider(guider, L, cfg):
    m, _ = guider
    H = 128
    u8 = (kps_inputs("v-kps", 1, L, H, H, seed=L) * 255).round().to(torch.uint8)
    x = u8.float() / 255.0
    pipe = _pipeline(guider=m)
    with torch.no_grad():
        feat = pipe.prepare_kps_feature(x, H, H, cfg)
        per_frame = torch.cat([m(x[:, :, j:j + 1].to(device="cuda", dtype=BF16)) for j in range(L)], 2)
        arrays = [u8[0, :, j].permute(1, 2, 0).numpy() for j in range(L)]
        from_arrays = pipe.prepare_kps_feature(arrays, H, H, cfg)
    assert feat.shape == (2 if cfg else 1, 320, L, H // 8, H // 8)
    assert _bits_equal(feat[-1:], per_frame)
    if cfg:
        assert bool((feat[:1].view(torch.int16) == 0).all()), "uncond half not exactly zero"
    assert _bits_equal(from_arrays, feat), "HWC uint8 arrays differ from the tensor input"


@pytest.mark.gpu
def test_projection_frames_are_independent(projection):
    p, _ = projection
    x = audio_inputs("jumpy", 300, seed=7).cuda()
    with torch.no_grad():
        full = p(x)
        for l in (0, 1, 2, 150, 298, 299):
            assert _bits_equal(p(x[l:l + 1]), full[l:l + 1]), f"frame {l}"


# ---- 6. pipeline hooks
@pytest.mark.gpu
def test_pipeline_hooks_against_fp64(guider, projection):
    m, gsd = guider
    p, psd = projection
    L, H = 20, 256
    g = _gen("hooks")
    states = (torch.randn(1, 53, 768, generator=g) * (0.2 + 2 * torch.rand(768, generator=g))).to(BF16).cuda()
    pipe = _pipeline(guider=m, projection=p, states=states)
    kps = kps_inputs("v-kps", 1, L, H, H, seed=20)
    with torch.no_grad():
        audio = pipe.prepare_audio_embeddings(torch.zeros(16000), L, 2, True)
        feat = pipe.prepare_kps_feature(kps, H, H, True)
        win64 = O.audio_frame_windows(states.double().cpu(), L).cuda()
        a_ref = O.audio_projection_forward(psd, AP, win64)
        a_eager = O.audio_projection_forward({k: v.to(BF16) for k, v in psd.items()}, AP,
                                             O.audio_frame_windows(states.cpu(), L).cuda())
        k_ref = torch.cat([_guider_ref(gsd, kps[:, :, i:i + 16].cuda(), F64) for i in range(0, L, 16)], 2)
        k_eager = torch.cat([_guider_ref(gsd, kps[:, :, i:i + 16].cuda(), BF16) for i in range(0, L, 16)], 2)
    assert audio.shape == (2, L, 5, 768) and feat.shape == (2, 320, L, H // 8, H // 8)
    assert bool((audio[0].view(torch.int16) == 0).all()) and bool((feat[0].view(torch.int16) == 0).all())
    fails = [_record("hook prepare_audio_embeddings L 20", _measure(audio[1], a_ref, a_ref),
                     _measure(a_eager, a_ref, a_ref), 1.0, bool(torch.isfinite(audio.float()).all())),
             _record("hook prepare_kps_feature L 20", _measure(feat[1:], k_ref, k_ref), _measure(k_eager, k_ref, k_ref),
                     1.0, bool(torch.isfinite(feat.float()).all()))]
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)
