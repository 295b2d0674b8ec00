"""Operator-level host wrappers over the C ABI (torch tensors in, raw pointers across the boundary).

Activations are bf16, channels-last token matrices ``[rows, C]`` (rows = (b f) h w); weights are bf16
``[N, K]`` (nn.Linear layout; conv weights repacked to ``[Cout, (ky kx cin)]``); biases fp32.
All launches go to torch's current CUDA stream, are asynchronous and CUDA-graph capturable."""
import ctypes
import os

import torch

from . import _ffi
from ._ffi import c_float, c_int, c_ll, check, ptr, stream_ptr

BF16 = torch.bfloat16


def _chk_bf16(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.dtype == BF16 and t.stride(-1) == 1, (t.dtype, t.device, t.stride())


def _chk_vectors(what, ld_mult, *ts):
    """The norm / activation kernels move 16-byte vectors and never check an address: every tensor handed to them must
    start 16-byte aligned and (2-D) have a row stride that is a multiple of ``ld_mult`` elements (8 bf16, 4 fp32)."""
    for t in ts:
        if t is not None and (t.data_ptr() % 16 or (t.dim() == 2 and t.stride(0) % ld_mult)):
            raise ValueError(f"{what}: operands must be 16-byte aligned with row strides that are multiples of {ld_mult}, "
                             f"got a {tuple(t.shape)} {t.dtype} view at byte offset {t.data_ptr() % 16} (mod 16), "
                             f"strides {t.stride()}")


def _chk_bias(bias, N, device, bias2=None, M=1, bias2_div=1):
    """The epilogue reads bias[n] and bias2[(m // bias2_div) * N + n] (n < N, m < M) as float2 from raw pointers: both must
    be fp32 on the output's device with unit column stride and 8-byte alignment, bias N entries, bias2 N columns and
    (M - 1) // bias2_div + 1 rows, with row stride N whenever more than one row is read (a strided column slice such as
    the per-block time embedding passes when one row serves every output row)."""
    for name, t in (("bias", bias), ("bias2", bias2)):
        if t is None:
            continue
        if t.dtype != torch.float32 or t.device != device or t.stride(-1) != 1 or t.data_ptr() % 8:
            raise ValueError(f"{name} must be fp32 on {device} with unit column stride and 8-byte alignment, got "
                             f"{t.dtype} on {t.device}, strides {t.stride()}")
    if bias is not None and (bias.dim() != 1 or bias.shape[0] != N):
        raise ValueError(f"bias must have shape ({N},), got {tuple(bias.shape)}")
    if bias2 is not None:
        if bias2_div < 1:
            raise ValueError(f"bias2_div must be >= 1, got {bias2_div}")
        rows = (M - 1) // bias2_div + 1
        b2 = bias2 if bias2.dim() == 2 else bias2.view(1, -1) if bias2.dim() == 1 else None
        if b2 is None or b2.shape[1] != N or b2.shape[0] < rows or (rows > 1 and b2.stride(0) != N):
            raise ValueError(f"bias2 must be [>= {rows}, {N}] with row stride {N} when more than one row is read "
                             f"(M = {M}, bias2_div = {bias2_div}), got shape {tuple(bias2.shape)} strides {bias2.stride()}")


def f32_arena(vectors, device):
    """All 1-D parameters of a model (biases, norm affine) as fp32 views into ONE buffer: one concatenation and two
    casts instead of a cast kernel per parameter.  Values are rounded to the model dtype first (what ``.to(bf16)`` does
    to the reference's parameters) and then widened; every view is 16-byte aligned (float4 loads in the epilogues)."""
    offs, parts, off = {}, [], 0
    for k, v in vectors.items():
        v = v.detach().reshape(-1)
        pad = (-v.numel()) % 4
        offs[k] = (off, v.numel())
        parts.append(torch.nn.functional.pad(v, (0, pad)) if pad else v)
        off += v.numel() + pad
    if not parts:
        return {}
    flat = torch.cat(parts).to(device=device, dtype=BF16).float()
    return {k: flat[o:o + n] for k, (o, n) in offs.items()}


def geglu_block_n(N):
    """wgmma N used for a GEGLU-fused GEMM with N = 2*inner accumulator columns (fixed at weight-packing time)."""
    for bn in (256, 128, 64):
        if N % bn == 0:
            return bn
    raise ValueError(f"GEGLU GEMM needs N % 64 == 0, got {N}")


def pack_geglu(w, bias, bn=None):
    """Reorder the rows of FeedForward.net.0.proj ([2*inner, K]: value rows then gate rows) so that every
    block_n-wide output tile holds block_n/2 value columns followed by the matching block_n/2 gate columns
    (block_n = bn, default geglu_block_n(N); gemm(geglu=True) needs the same block_n)."""
    N = w.shape[0]
    bn = bn or geglu_block_n(N)
    inner, hb = N // 2, bn // 2
    idx = torch.arange(N, device=w.device).view(N // bn, 2, hb)
    t = torch.arange(N // bn, device=w.device).view(-1, 1)
    j = torch.arange(hb, device=w.device).view(1, -1)
    idx = torch.stack([t * hb + j, inner + t * hb + j], 1).reshape(-1)
    return w[idx].contiguous(), (None if bias is None else bias[idx].contiguous()), bn


def gemm(a, w, bias=None, *, a2=None, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None, block_n=0,
         out_f32=False, geglu=False):
    """out = (concat(a, a2) @ w.T + bias + bias2[row // bias2_div]) * scale + residual  (bf16, or fp32 if out_f32).
    geglu=True: w/bias packed by pack_geglu (at block_n, default geglu_block_n(N)); out[:, j] = (v_j + b) * gelu(g_j + b)
    with N/2 columns."""
    _chk_bf16(a, w, a2, residual, None if out_f32 else out)
    M, K1 = a.shape
    K2 = 0 if a2 is None else a2.shape[1]
    N = w.shape[0]
    assert w.shape[1] == K1 + K2
    _chk_bias(bias, N, a.device, bias2, M, bias2_div)
    if geglu and not block_n:
        block_n = geglu_block_n(N)
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), device=a.device, dtype=torch.float32 if out_f32 else BF16)
    check(_ffi.lib().vx_gemm_bf16(
        ptr(a), c_ll(a.stride(0)), c_int(K1), ptr(a2), c_ll(0 if a2 is None else a2.stride(0)), c_int(K2),
        ptr(w), c_ll(w.stride(0)), c_int(M), c_int(N), ptr(bias), ptr(bias2), c_int(bias2_div), c_float(scale),
        ptr(residual), c_ll(0 if residual is None else residual.stride(0)), ptr(out), c_ll(out.stride(0)),
        c_int(2 if geglu else int(out_f32)), c_int(block_n), stream_ptr()), "vx_gemm_bf16")
    return out


# ---- FP8 (e4m3) operands with per-row / per-output-channel scales (opt-in: UNet3DConditionModel.enable_fp8_linear)
E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def quantize_fp8_weight(w):
    """[N, K] weight -> (float8_e4m3fn codes [N, K], fp32 scale [N]): scale[n] = amax_k |w[n, k]| / 448 (1 for an all-zero
    row), codes = clamp(w / scale, +-448) cast to e4m3 (round to nearest even; torch's cast does not saturate, hence the
    clamp).  Per output channel, so a fused q|k|v weight carries the concatenated scales of q, k and v, and a weight packed
    by pack_geglu gets codes and scales in its (value | gate) tile order."""
    wf = w.float()
    amax = wf.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    codes = (wf / scale[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3).contiguous()
    return codes, scale.contiguous()


def gemm_fp8(a, a_scale, w, w_scale, bias=None, *, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None,
             block_n=0, geglu=False):
    """gemm() on e4m3 operands: out = epilogue(a_scale[m] * w_scale[n] * (a @ w.T)[m, n]) in bf16.  a [M, K] / w [N, K]
    float8_e4m3fn (K a multiple of 16), a_scale [M] / w_scale [N] fp32; bias, bias2, scale, residual and geglu (w, w_scale
    and bias packed by pack_geglu) as in gemm()."""
    for t in (a, w):
        assert t.is_cuda and t.dtype == E4M3 and t.stride(-1) == 1, (t.dtype, t.device, t.stride())
    _chk_bf16(residual, out)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K
    for name, t, n in (("a_scale", a_scale, M), ("w_scale", w_scale, N)):
        if t.dtype != torch.float32 or t.device != a.device or not t.is_contiguous() or t.shape != (n,) or t.data_ptr() % 8:
            raise ValueError(f"{name} must be a contiguous fp32 [{n}] vector on {a.device}, got {t.dtype} {tuple(t.shape)}")
    _chk_bias(bias, N, a.device, bias2, M, bias2_div)
    if geglu and not block_n:
        block_n = geglu_block_n(N)
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), device=a.device, dtype=BF16)
    check(_ffi.lib().vx_gemm_fp8(
        ptr(a), c_ll(a.stride(0)), ptr(a_scale), c_int(K), ptr(w), c_ll(w.stride(0)), ptr(w_scale), c_int(M), c_int(N),
        ptr(bias), ptr(bias2), c_int(bias2_div), c_float(scale), ptr(residual), c_ll(0 if residual is None else residual.stride(0)),
        ptr(out), c_ll(out.stride(0)), c_int(int(geglu)), c_int(block_n), stream_ptr()), "vx_gemm_fp8")
    return out


# ---- LayerNorm folded into the consumer GEMM (experiment; the engine uses it only under VX_LN_FOLD=1)
def row_stats(x, eps=1e-5, out=None):
    """(mean, rstd) of every row of x [rows, C] bf16 -> fp32 [rows, 2]."""
    _chk_vectors("row_stats", 8, x)
    _chk_bf16(x)
    rows, C = x.shape
    if out is None:
        out = torch.empty((rows, 2), device=x.device, dtype=torch.float32)
    check(_ffi.lib().vx_row_stats(ptr(x), c_ll(x.stride(0)), c_ll(rows), c_int(C), c_float(eps), ptr(out), stream_ptr()),
          "vx_row_stats")
    return out


def fold_layernorm(w, bias, gamma, beta, geglu=False):
    """LayerNorm(x) @ w.T + bias  ==  rstd * (x @ wf.T - mean * colsum) + bf   with
    wf = bf16(w * gamma), colsum = sum_k wf, bf = w @ beta + bias.  w bf16 [N, K]; gamma/beta/bias fp32.
    geglu=True additionally applies pack_geglu's row order to all three.
    colsum must be the sum of the ROUNDED wf: then mean * colsum cancels the uncentred part of x @ wf.T exactly and the
    weight rounding stays a centred 2^-9 r sum |x_k - mean| |gamma_k w_k| (half the default path's LayerNorm output
    rounding).  What the fold still pays is the uncentred fp32 accumulation, (K + 2) 2^-22 (|mean| / sigma) sum |wf_k| at
    worst: tests/test_lnfold_bounds_gpu.py holds the fused GEMMs to the default path's accuracy bound for rows with
    |mean| / sigma <= R(K) = 0.8 * 2^12 / (K + 2) (10.2 at K = 320, 2.6 at K = 1280).  Beyond that, and on near-constant
    rows, there is no such guarantee; the measured error stayed at the default path's up to |mean| / sigma ~ 64."""
    wf = (w.float() * gamma.float()[None, :]).to(BF16)
    bf = w.float() @ beta.float()
    if bias is not None:
        bf = bf + bias.float()
    if geglu:
        wf, bf, _ = pack_geglu(wf, bf)
    return wf.contiguous(), wf.float().sum(1).contiguous(), bf.contiguous()


def gemm_lnfold(a, wf, stats, colsum, bias, *, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None, geglu=False):
    """out = rstd * (a @ wf.T - mean * colsum) + bias (+ bias2[row // bias2_div]) (* scale + residual | GEGLU)."""
    _chk_bf16(a, wf, residual, out)
    M, K = a.shape
    N = wf.shape[0]
    assert wf.shape[1] == K and stats.shape == (M, 2) and colsum.shape == (N,)
    _chk_bias(bias, N, a.device, bias2, M, bias2_div)
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), device=a.device, dtype=BF16)
    check(_ffi.lib().vx_gemm_lnfold_bf16(
        ptr(a), c_ll(a.stride(0)), c_int(K), ptr(wf), c_ll(wf.stride(0)), c_int(M), c_int(N), ptr(stats), ptr(colsum),
        ptr(bias), ptr(bias2), c_int(bias2_div), c_float(scale), ptr(residual),
        c_ll(0 if residual is None else residual.stride(0)), ptr(out), c_ll(out.stride(0)), c_int(int(geglu)),
        c_int(geglu_block_n(N) if geglu else 0), stream_ptr()), "vx_gemm_lnfold_bf16")
    return out


def rowsum_slots(N):
    """Upper bound of the 2 * ceil(N / block_n) partial sums per row vx_gemm_rowsums_bf16 may write (block_n >= 32)."""
    return 2 * ((N + 31) // 32)


def gemm_rowsums(a, w, bias=None, *, a2=None, scale=1.0, residual=None, out=None):
    """ops.gemm (linear epilogue, bf16) that also returns the LayerNorm hand-over of its output: (out, parts, nparts) with
    parts fp32 [rowsum_slots(N), M, 2] = per-row partial (sum, sum of squares) of the rounded outputs in slots < nparts."""
    _chk_bf16(a, w, a2, residual, out)
    M, K1 = a.shape
    K2 = 0 if a2 is None else a2.shape[1]
    N = w.shape[0]
    assert w.shape[1] == K1 + K2 and N // 32 * 2 >= 2
    _chk_bias(bias, N, a.device)
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=BF16)
    cap = rowsum_slots(N)
    parts = torch.empty((cap, M, 2), device=a.device, dtype=torch.float32)
    nparts = c_int(0)
    check(_ffi.lib().vx_gemm_rowsums_bf16(
        ptr(a), c_ll(a.stride(0)), c_int(K1), ptr(a2), c_ll(0 if a2 is None else a2.stride(0)), c_int(K2),
        ptr(w), c_ll(w.stride(0)), c_int(M), c_int(N), ptr(bias), ptr(None), c_int(1), c_float(scale),
        ptr(residual), c_ll(0 if residual is None else residual.stride(0)), ptr(out), c_ll(out.stride(0)),
        c_int(0), ptr(parts), c_ll(M), c_int(cap), ctypes.byref(nparts), stream_ptr()), "vx_gemm_rowsums_bf16")
    assert 0 < nparts.value <= cap, nparts.value
    return out, parts, nparts.value


def gemm_lnparts(a, wf, parts, nparts, colsum, bias, eps=1e-5, *, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None,
                 geglu=False):
    """gemm_lnfold with the row statistics of `a` taken from its producer's partial sums (gemm_rowsums)."""
    _chk_bf16(a, wf, residual, out)
    M, K = a.shape
    N = wf.shape[0]
    assert wf.shape[1] == K and parts.shape[1:] == (M, 2) and 0 < nparts <= parts.shape[0] and colsum.shape == (N,)
    _chk_bias(bias, N, a.device, bias2, M, bias2_div)
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), device=a.device, dtype=BF16)
    check(_ffi.lib().vx_gemm_lnparts_bf16(
        ptr(a), c_ll(a.stride(0)), c_int(K), ptr(wf), c_ll(wf.stride(0)), c_int(M), c_int(N), ptr(parts), c_ll(M),
        c_int(nparts), c_float(eps), ptr(colsum), ptr(bias), ptr(bias2), c_int(bias2_div), c_float(scale), ptr(residual),
        c_ll(0 if residual is None else residual.stride(0)), ptr(out), c_ll(out.stride(0)), c_int(int(geglu)),
        c_int(geglu_block_n(N) if geglu else 0), stream_ptr()), "vx_gemm_lnparts_bf16")
    return out


def conv3x3(x, w, bias=None, *, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None, block_n=0):
    """x: NHWC bf16 [NB,H,W,C]; w: [Cout, 9*C]; returns [NB*H*W, Cout] (= NHWC)."""
    _chk_bf16(x, w, residual, out)
    assert x.is_contiguous()
    NB, H, W, C = x.shape
    Cout = w.shape[0]
    assert w.shape[1] == 9 * C
    _chk_bias(bias, Cout, x.device, bias2, NB * H * W, bias2_div)
    if out is None:
        out = torch.empty((NB * H * W, Cout), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_conv3x3_bf16(
        ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), ptr(w), c_int(Cout), ptr(bias), ptr(bias2),
        c_int(bias2_div), c_float(scale), ptr(residual), c_ll(0 if residual is None else residual.stride(0)),
        ptr(out), c_ll(out.stride(0)), c_int(block_n), stream_ptr()), "vx_conv3x3_bf16")
    return out


CONV_S2_TMA = os.environ.get("VX_CONV_S2", "1") != "0"   # A/B switch: 0 = im2col + GEMM (the round-1 path)


def downsample_conv(x, NB, H, W, w, bias, pad_lo=1):
    """Stride-2 3x3 conv of the [NB*H*W, C] token matrix -> [NB*(H/2)*(W/2), Cout]."""
    if CONV_S2_TMA and x.shape[1] % 64 == 0:
        return conv3x3_s2(x.view(NB, H, W, x.shape[1]), w, bias, pad_lo=pad_lo)
    col = im2col_s2(x, NB, H, W) if pad_lo == 1 else im2col3x3(x, NB, H, W, stride=2, pad_lo=0)
    return gemm(col, w, bias)


def conv3x3_s2(x, w, bias=None, *, pad_lo=1, out=None, block_n=0):
    """3x3 conv, stride 2, on the tensor cores straight from the NHWC input (TMA traversal stride 2: no im2col tensor).
    x: NHWC bf16 [NB,H,W,C], H and W even; w: [Cout, 9*C]; returns [NB*(H/2)*(W/2), Cout].  pad_lo=1: padding 1 all round
    (UNet downsamplers); pad_lo=0: pad (0,1,0,1) (VAE encoder downsamplers)."""
    _chk_bf16(x, w, out)
    assert x.is_contiguous()
    NB, H, W, C = x.shape
    Cout = w.shape[0]
    assert w.shape[1] == 9 * C and H % 2 == 0 and W % 2 == 0
    _chk_bias(bias, Cout, x.device)
    if out is None:
        out = torch.empty((NB * (H // 2) * (W // 2), Cout), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_conv3x3s2_bf16(
        ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), ptr(w), c_int(Cout), ptr(bias), c_int(pad_lo), ptr(out),
        c_ll(out.stride(0)), c_int(block_n), stream_ptr()), "vx_conv3x3s2_bf16")
    return out


def pack_upconv_weight(w):
    """(Cout, Cin, 3, 3) conv weight of an `nearest-2x upsample -> conv3x3` pair -> [4*Cout, 4*Cin] bf16 for
    vx_upconv3x3_bf16: block (py, px) holds the 2x2 kernel seen by output pixels (2i+py, 2j+px); tap a (b) of that kernel
    reads input row i + py - 1 + a (column j + px - 1 + b) and is the fp32 sum of the 3x3 rows (columns) that fall on it:
    py = 0: a=0 <- ky {0}, a=1 <- ky {1,2};  py = 1: a=0 <- ky {0,1}, a=1 <- ky {2}.  K order (a, b, cin)."""
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    wf = w.float()
    blocks = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for a in (0, 1):
                for b in (0, 1):
                    acc = 0
                    for ky in groups[py][a]:
                        for kx in groups[px][b]:
                            acc = acc + wf[:, :, ky, kx]
                    taps.append(acc)                                  # (Cout, Cin)
            blocks.append(torch.stack(taps, 1).reshape(w.shape[0], -1))   # (Cout, 4*Cin), K = (tap, cin)
    return torch.cat(blocks, 0).to(BF16).contiguous()


def upconv3x3(x, w4, bias, out=None, block_n=0):
    """x: NHWC bf16 [NB,H,W,C]; w4 from pack_upconv_weight; returns conv3x3(upsample2x(x)) as [NB*2H*2W, Cout]."""
    _chk_bf16(x, w4, out)
    assert x.is_contiguous()
    NB, H, W, C = x.shape
    Cout = w4.shape[0] // 4
    assert w4.shape[1] == 4 * C
    _chk_bias(bias, Cout, x.device)
    if out is None:
        out = torch.empty((NB * 4 * H * W, Cout), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_upconv3x3_bf16(ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), ptr(w4), c_int(Cout), ptr(bias),
                                       ptr(out), c_ll(out.stride(0)), c_int(block_n), stream_ptr()), "vx_upconv3x3_bf16")
    return out


def pack_conv3x3_weight(w):
    """(Cout, Cin, 3, 3) -> [Cout, (ky kx cin)] bf16, the K order the implicit-GEMM producer walks."""
    co, ci, kh, kw = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous()


# ----------------------------------------------------------------------------- bring-up probes
def probe_umma(a_img, b_img, lboA, sboA, layA, lboB, sboB, layB, a_mn, b_mn, N, ksteps, a_step, b_step):
    out = torch.empty((128, N), device=a_img.device, dtype=torch.float32)
    check(_ffi.lib().vx_probe_umma(ptr(a_img), c_int(a_img.numel()), ptr(b_img), c_int(b_img.numel()),
                                   ctypes.c_uint(lboA), ctypes.c_uint(sboA), ctypes.c_uint(layA),
                                   ctypes.c_uint(lboB), ctypes.c_uint(sboB), ctypes.c_uint(layB), c_int(a_mn),
                                   c_int(b_mn), c_int(N), c_int(ksteps), c_int(a_step), c_int(b_step), ptr(out),
                                   stream_ptr()), "vx_probe_umma")
    return out


def probe_tma(base, dims, strides_bytes, box, swizzle, coords, nbytes):
    rank = len(dims)
    out = torch.empty(nbytes, device=base.device, dtype=torch.uint8)
    U64 = ctypes.c_ulonglong * 5
    U32 = ctypes.c_uint * 5
    I32 = ctypes.c_int * 5
    pad = lambda x, n: list(x) + [0] * (n - len(x))
    check(_ffi.lib().vx_probe_tma(ptr(base), c_int(rank), U64(*pad(dims, 5)), U64(*pad(strides_bytes, 5)),
                                  U32(*pad(box, 5)), c_int(swizzle), I32(*pad(coords, 5)), c_int(nbytes), ptr(out),
                                  stream_ptr()), "vx_probe_tma")
    return out


# ----------------------------------------------------------------------------- attention
def flash_attention(q, k, v, heads, Nq, Nk, kv_div=1, out=None):
    """q: [Bq*Nq, >=heads*hd] (row stride arbitrary), k/v: [Bkv*Nk, ...]; returns [Bq*Nq, heads*hd]."""
    _chk_bf16(q, k, v, out)
    C = q.shape[1]
    hd = C // heads
    Bq = q.shape[0] // Nq
    Bkv = k.shape[0] // Nk
    if out is None:
        out = torch.empty((q.shape[0], C), device=q.device, dtype=BF16)
    check(_ffi.lib().vx_flash_attention(ptr(q), c_ll(q.stride(0)), ptr(k), c_ll(k.stride(0)), ptr(v),
                                        c_ll(v.stride(0)), ptr(out), c_ll(out.stride(0)), c_int(Bq), c_int(Nq),
                                        c_int(Bkv), c_int(Nk), c_int(heads), c_int(hd), c_int(kv_div), stream_ptr()),
          "vx_flash_attention")
    return out


def temporal_attention(q, k, v, b, f, HW, heads, out=None):
    """q/k/v: [(b f HW), C] column slices sharing one row stride; attention over f per (b, pixel, head)."""
    _chk_bf16(q, k, v, out)
    assert q.stride(0) == k.stride(0) == v.stride(0)
    C = q.shape[1]
    if out is None:
        out = torch.empty((q.shape[0], C), device=q.device, dtype=BF16)
    check(_ffi.lib().vx_temporal_attention(ptr(q), ptr(k), ptr(v), c_ll(q.stride(0)), ptr(out), c_ll(out.stride(0)),
                                           c_int(b), c_int(f), c_int(HW), c_int(heads), c_int(C // heads),
                                           stream_ptr()), "vx_temporal_attention")
    return out


def smallkv_attention(q, k, v, rows_per_frame, heads, Lk, out=None):
    """q: [rows, C]; k/v: [frames*Lk, C] (shared row stride)."""
    _chk_bf16(q, k, v, out)
    assert k.stride(0) == v.stride(0)
    C = q.shape[1]
    if out is None:
        out = torch.empty((q.shape[0], C), device=q.device, dtype=BF16)
    check(_ffi.lib().vx_smallkv_attention(ptr(q), c_ll(q.stride(0)), ptr(k), ptr(v), c_ll(k.stride(0)), ptr(out),
                                          c_ll(out.stride(0)), c_ll(q.shape[0]), c_int(rows_per_frame), c_int(heads),
                                          c_int(C // heads), c_int(Lk), stream_ptr()), "vx_smallkv_attention")
    return out


LN_GEMM_MAX_K = 512   # vx_gemm_ln_bf16 keeps the whole 128-row x K tile in shared memory


def gemm_ln(a, wf, colsum, bias, eps=1e-5, *, bias2=None, bias2_div=1, scale=1.0, residual=None, out=None, geglu=False):
    """LayerNorm(a) @ W.T + b in one kernel (fold_layernorm's wf / colsum / bias; row statistics computed in the kernel from
    the shared-memory resident row tile): out = rstd * (a @ wf.T - mean * colsum) + bias (+ bias2[row // bias2_div])
    (* scale + residual | GEGLU).  K = a.shape[1] must be a multiple of 64 and <= LN_GEMM_MAX_K."""
    _chk_bf16(a, wf, residual, out)
    M, K = a.shape
    N = wf.shape[0]
    assert wf.shape[1] == K and colsum.shape == (N,) and K % 64 == 0 and K <= LN_GEMM_MAX_K
    _chk_bias(bias, N, a.device, bias2, M, bias2_div)
    if out is None:
        out = torch.empty((M, N // 2 if geglu else N), device=a.device, dtype=BF16)
    check(_ffi.lib().vx_gemm_ln_bf16(
        ptr(a), c_ll(a.stride(0)), c_int(K), ptr(wf), c_ll(wf.stride(0)), c_int(M), c_int(N), ptr(colsum), ptr(bias),
        c_float(eps), ptr(bias2), c_int(bias2_div), c_float(scale), ptr(residual),
        c_ll(0 if residual is None else residual.stride(0)), ptr(out), c_ll(out.stride(0)), c_int(int(geglu)),
        c_int(geglu_block_n(N) if geglu else 0), stream_ptr()), "vx_gemm_ln_bf16")
    return out


# ----------------------------------------------------------------------------- norms / activations
_GN_CAP = {}


def _gn_S(NB, HW, C=0):
    """Pixel chunks per frame: NB * S CTAs = ONE wave of what the device actually keeps resident for this channel count
    (occupancy query in the library), so both GroupNorm passes run without a ragged second wave and the one-launch
    kernel's rendezvous is safe."""
    cap = _GN_CAP.get(C)
    if cap is None:
        cap = (_ffi.lib().vx_groupnorm_capacity(c_int(C)) if C
               else torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 4)
        _GN_CAP[C] = cap = max(int(cap), 1)
    s = max(1, min(HW // 32, cap // max(NB, 1)))
    return max(1, min(s, 64))


_GN_FUSED = os.environ.get("VX_GN_FUSED", "1") != "0"
_GN_CLUSTER = os.environ.get("VX_GN_CLUSTER", "1") != "0"   # cluster-resident GroupNorm for small frames (0: A/B switch)
_GN_COUNTERS = {}


def _gn_counters(device, NB):
    """int32 [2 * NB] rendezvous counters of the one-launch GroupNorm, zeroed once (the kernel recycles them)."""
    key = (device.type, device.index)
    t = _GN_COUNTERS.get(key)
    if t is None or t.numel() < 2 * NB:
        t = torch.zeros(max(2 * NB, 1024), device=device, dtype=torch.int32)
        _GN_COUNTERS[key] = t
    return t


def groupnorm(x1, NB, HW, gamma, beta, eps, silu, x2=None, groups=32, out=None, ws=None):
    """Per-frame GroupNorm (+SiLU) of the channel-concatenation [x1 | x2]; x*: [NB*HW, C*] bf16.

    VX_GN_FRAMES=n (experiment, default off) runs the statistics and the apply kernel on groups of n frames
    back to back so that the second read of a group is served by the L2 instead of HBM."""
    grp = int(os.environ.get("VX_GN_FRAMES", "0"))
    if 0 < grp < NB:
        return _groupnorm_grouped(x1, NB, HW, gamma, beta, eps, silu, x2, groups, out, grp)
    _chk_vectors("groupnorm", 8, x1, x2, out)
    _chk_bf16(x1, x2, out)
    C1 = x1.shape[1]
    C2 = 0 if x2 is None else x2.shape[1]
    if out is None:
        out = torch.empty((NB * HW, C1 + C2), device=x1.device, dtype=BF16)
    L = _ffi.lib()
    ld2 = c_ll(0 if x2 is None else x2.stride(0))
    if _GN_CLUSTER:                     # small frames: resident in a cluster's shared memory, one pass over HBM
        rc = L.vx_groupnorm_cluster(ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), ld2, c_int(C2), c_int(NB), c_int(HW),
                                    c_int(groups), ptr(gamma), ptr(beta), c_float(eps), c_int(int(silu)), ptr(out),
                                    c_ll(out.stride(0)), stream_ptr())
        if rc != 2:                     # 2 = the frame does not fit a cluster
            check(rc, "vx_groupnorm_cluster")
            return out
    S = _gn_S(NB, HW, C1 + C2)
    if ws is None:
        ws = torch.empty(NB * S * groups * 3, device=x1.device, dtype=torch.float32)
    if _GN_FUSED:
        rc = L.vx_groupnorm_fused(ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), ld2, c_int(C2), c_int(NB), c_int(HW),
                                  c_int(groups), c_int(S), ptr(ws), ptr(_gn_counters(x1.device, NB)), ptr(gamma), ptr(beta),
                                  c_float(eps), c_int(int(silu)), ptr(out), c_ll(out.stride(0)), stream_ptr())
        if rc != 2:                     # 2 = grid cannot be co-resident: fall through to the two-kernel pair
            check(rc, "vx_groupnorm_fused")
            return out
    check(L.vx_groupnorm_stats(ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), ld2, c_int(C2), c_int(NB), c_int(HW),
                               c_int(groups), c_int(S), ptr(ws), stream_ptr()), "vx_groupnorm_stats")
    check(L.vx_groupnorm_apply(ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), ld2, c_int(C2), c_int(NB), c_int(HW),
                               c_int(groups), c_int(S), ptr(ws), ptr(gamma), ptr(beta), c_float(eps), c_int(int(silu)),
                               ptr(out), c_ll(out.stride(0)), stream_ptr()), "vx_groupnorm_apply")
    return out


def _groupnorm_grouped(x1, NB, HW, gamma, beta, eps, silu, x2, groups, out, grp):
    _chk_vectors("groupnorm", 8, x1, x2, out)
    _chk_bf16(x1, x2, out)
    C1 = x1.shape[1]
    C2 = 0 if x2 is None else x2.shape[1]
    if out is None:
        out = torch.empty((NB * HW, C1 + C2), device=x1.device, dtype=BF16)
    L = _ffi.lib()
    for n0 in range(0, NB, grp):
        nb = min(grp, NB - n0)
        r0, r1 = n0 * HW, (n0 + nb) * HW
        a1 = x1[r0:r1]
        a2 = None if x2 is None else x2[r0:r1]
        o = out[r0:r1]
        S = _gn_S(nb, HW, C1 + C2)
        w = torch.empty(nb * S * groups * 3, device=x1.device, dtype=torch.float32)
        ld2 = c_ll(0 if a2 is None else a2.stride(0))
        check(L.vx_groupnorm_stats(ptr(a1), c_ll(a1.stride(0)), c_int(C1), ptr(a2), ld2, c_int(C2), c_int(nb), c_int(HW),
                                   c_int(groups), c_int(S), ptr(w), stream_ptr()), "vx_groupnorm_stats")
        check(L.vx_groupnorm_apply(ptr(a1), c_ll(a1.stride(0)), c_int(C1), ptr(a2), ld2, c_int(C2), c_int(nb), c_int(HW),
                                   c_int(groups), c_int(S), ptr(w), ptr(gamma), ptr(beta), c_float(eps), c_int(int(silu)),
                                   ptr(o), c_ll(out.stride(0)), stream_ptr()), "vx_groupnorm_apply")
    return out


def layernorm(x, gamma, beta, eps=1e-5, pe=None, rows_per_frame=0, out=None):
    _chk_vectors("layernorm", 8, x, out, gamma, beta, pe)
    _chk_bf16(x, out)
    rows, C = x.shape
    if out is None:
        out = torch.empty((rows, C), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_layernorm(ptr(x), c_ll(x.stride(0)), c_ll(rows), c_int(C), ptr(gamma), ptr(beta),
                                  c_float(eps), ptr(pe), c_int(rows_per_frame), c_int(0 if pe is None else pe.shape[0]),
                                  ptr(out), c_ll(out.stride(0)), stream_ptr()), "vx_layernorm")
    return out


def layernorm_fp8(x, gamma, beta, eps=1e-5, pe=None, rows_per_frame=0, out=None, row_scale=None):
    """layernorm() as the A operand of gemm_fp8: (float8_e4m3fn codes [rows, C], fp32 row_scale [rows]) with
    codes * row_scale ~ LayerNorm(x) [+ pe] computed in fp32, row_scale = amax(|row|) / 448 (1 for an all-zero row)."""
    _chk_vectors("layernorm_fp8", 8, x)
    _chk_bf16(x)
    rows, C = x.shape
    if out is None:
        out = torch.empty((rows, C), device=x.device, dtype=E4M3)
    if row_scale is None:
        row_scale = torch.empty((rows,), device=x.device, dtype=torch.float32)
    # the kernel stores eight codes at a time (8-byte aligned rows) and reads gamma / beta / pe as float4
    if (out.dtype != E4M3 or out.device != x.device or out.stride(-1) != 1 or out.shape != (rows, C)
            or out.data_ptr() % 8 or out.stride(0) % 8):
        raise ValueError(f"out must be a [{rows}, {C}] float8_e4m3fn view on {x.device} with unit column stride and 8-byte "
                         f"aligned rows, got {out.dtype} {tuple(out.shape)} strides {out.stride()} at offset {out.data_ptr() % 8}")
    if row_scale.dtype != torch.float32 or row_scale.device != x.device or not row_scale.is_contiguous() \
            or row_scale.numel() != rows:
        raise ValueError(f"row_scale must be a contiguous fp32 [{rows}] vector on {x.device}")
    for name, t, n in (("gamma", gamma, C), ("beta", beta, C), ("pe", pe, None)):
        if t is None and name == "pe":
            continue
        if (t.dtype != torch.float32 or t.device != x.device or not t.is_contiguous() or t.data_ptr() % 16
                or t.shape[-1] != C or (n is not None and t.numel() != n)):
            raise ValueError(f"{name} must be contiguous fp32 on {x.device}, 16-byte aligned, with {C} columns; got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
    check(_ffi.lib().vx_layernorm_fp8(ptr(x), c_ll(x.stride(0)), c_ll(rows), c_int(C), ptr(gamma), ptr(beta),
                                      c_float(eps), ptr(pe), c_int(rows_per_frame), c_int(0 if pe is None else pe.shape[0]),
                                      ptr(out), c_ll(out.stride(0)), ptr(row_scale), stream_ptr()), "vx_layernorm_fp8")
    return out, row_scale


def geglu(x, out=None):
    _chk_vectors("geglu", 8, x, out)
    _chk_bf16(x, out)
    rows, two = x.shape
    inner = two // 2
    if out is None:
        out = torch.empty((rows, inner), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_geglu(ptr(x), c_ll(x.stride(0)), c_ll(rows), c_int(inner), ptr(out), c_ll(out.stride(0)),
                              stream_ptr()), "vx_geglu")
    return out


# ----------------------------------------------------------------------------- misc
def conv_in(x, w, bias, Cout, addend=None, add_frame=None, out=None, pre_scale=1.0, pre_w=None, pre_b=None):
    """x: planar bf16 (n, c, h, w) given as a 4-D tensor whose (h, w) plane is contiguous.
    Optional per-pixel pre-transform  v -> bf16(pre_w @ bf16(pre_scale * v) + pre_b)  (VAE: 1/0.18215 scaling and
    the 1x1 post_quant_conv) applied to in-bounds pixels before the 3x3 taps."""
    assert x.dtype == BF16 and x.stride(3) == 1 and x.stride(2) == x.shape[3]
    NB, Cin, H, W = x.shape
    if out is None:
        out = torch.empty((NB * H * W, Cout), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_conv_in(ptr(x), c_ll(x.stride(0)), c_ll(x.stride(1)), c_int(NB), c_int(H), c_int(W), c_int(Cin),
                                c_int(Cout), ptr(w), ptr(bias), ptr(addend), ptr(add_frame),
                                c_ll(0 if addend is None else addend.stride(0)), c_float(pre_scale), ptr(pre_w), ptr(pre_b),
                                ptr(out), c_ll(out.stride(0)), stream_ptr()), "vx_conv_in")
    return out


def conv_out(x, NB, H, W, w, bias, out, post=False):
    """x: NHWC [NB*H*W, C] bf16; w fp32 [Cout, 9, C]; out planar 4-D (n, co, h, w) bf16 or fp32."""
    _chk_bf16(x)
    assert out.stride(3) == 1 and out.stride(2) == W
    Cout = w.shape[0]
    check(_ffi.lib().vx_conv_out(ptr(x), c_ll(x.stride(0)), c_int(NB), c_int(H), c_int(W), c_int(x.shape[1]), c_int(Cout),
                                 ptr(w), ptr(bias), ptr(out), c_ll(out.stride(0)), c_ll(out.stride(1)),
                                 c_int(int(out.dtype == torch.float32)), c_int(int(post)), stream_ptr()), "vx_conv_out")
    return out


def im2col_s2(x, NB, H, W, out=None):
    _chk_bf16(x)
    C = x.shape[-1]
    if out is None:
        out = torch.empty((NB * (H // 2) * (W // 2), 9 * C), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_im2col_s2(ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), ptr(out), stream_ptr()), "vx_im2col_s2")
    return out


def upsample2x(x, NB, H, W, out=None):
    _chk_bf16(x)
    C = x.shape[-1]
    if out is None:
        out = torch.empty((NB * 4 * H * W, C), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_upsample2x(ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), ptr(out), stream_ptr()), "vx_upsample2x")
    return out


def skinny_linear(x, w, bias, act_in=False, act_out=False, out=None):
    assert x.dtype == torch.float32 and w.dtype == BF16 and x.is_contiguous() and w.is_contiguous()
    rows, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((rows, N), device=x.device, dtype=torch.float32)
    check(_ffi.lib().vx_skinny_linear(ptr(x), c_int(rows), c_int(K), ptr(w), ptr(bias), c_int(N), c_int(int(act_in)),
                                      c_int(int(act_out)), ptr(out), stream_ptr()), "vx_skinny_linear")
    return out


def timestep_embed(t, dim, out=None):
    assert t.dtype == torch.float32
    if out is None:
        out = torch.empty((t.shape[0], dim), device=t.device, dtype=torch.float32)
    check(_ffi.lib().vx_timestep_embed(ptr(t), c_int(t.shape[0]), c_int(dim), ptr(out), stream_ptr()), "vx_timestep_embed")
    return out


def cfg_overlap_accumulate(noise, f, hw, L, do_cfg, win, count, guidance, acc):
    check(_ffi.lib().vx_cfg_overlap_accumulate(ptr(noise), c_int(f), c_int(hw), c_int(L), c_int(int(do_cfg)), ptr(win),
                                               ptr(count), c_float(guidance), ptr(acc), stream_ptr()),
          "vx_cfg_overlap_accumulate")


def cfg_overlap_accumulate_n(noise, n, f, hw, L, do_cfg, win, count, guidance, acc):
    """cfg_overlap_accumulate for the n samples of one window: noise ((b n f),4,h,w) as [u s0..s(n-1) | c s0..s(n-1)],
    acc fp32 (n, 4, L, hw)."""
    assert noise.is_contiguous() and acc.is_contiguous() and acc.dtype == torch.float32
    assert noise.numel() == (2 if do_cfg else 1) * n * f * 4 * hw and acc.numel() == n * 4 * L * hw
    check(_ffi.lib().vx_cfg_overlap_accumulate_n(ptr(noise), c_int(n), c_int(f), c_int(hw), c_int(L), c_int(int(do_cfg)),
                                                 ptr(win), ptr(count), c_float(guidance), ptr(acc), stream_ptr()),
          "vx_cfg_overlap_accumulate_n")


def ddim_step(latents, acc, sqrt_a, sqrt_1ma, sqrt_aprev, sqrt_1maprev):
    check(_ffi.lib().vx_ddim_step(ptr(latents), ptr(acc), c_ll(latents.numel()), c_float(sqrt_a), c_float(sqrt_1ma),
                                  c_float(sqrt_aprev), c_float(sqrt_1maprev), stream_ptr()), "vx_ddim_step")


def ddim_step_eta(latents, acc, noise, sqrt_a, sqrt_1ma, sqrt_aprev, c_dir, sigma):
    """Stochastic DDIM step on all elements of latents bf16 (n,4,L,...): ``ddim_step`` with c_dir for sqrt(1-a_prev),
    plus bf16(sigma * noise); noise fp32 with the layout of latents (``scheduler.ddim_coefficients_eta``)."""
    if not (latents.dtype == BF16 and acc.dtype == torch.float32 and noise.dtype == torch.float32):
        raise ValueError(f"ddim_step_eta: latents bf16 / acc fp32 / noise fp32, got {latents.dtype} / {acc.dtype} / "
                         f"{noise.dtype}")
    if not (latents.is_contiguous() and acc.is_contiguous() and noise.is_contiguous()
            and acc.numel() == latents.numel() == noise.numel() and latents.device == acc.device == noise.device):
        raise ValueError(f"ddim_step_eta: latents {tuple(latents.shape)}, acc {tuple(acc.shape)} and noise "
                         f"{tuple(noise.shape)} must be contiguous tensors of equal size on one device")
    check(_ffi.lib().vx_ddim_step_eta(ptr(latents), ptr(acc), ptr(noise), c_ll(latents.numel()), c_float(sqrt_a),
                                      c_float(sqrt_1ma), c_float(sqrt_aprev), c_float(c_dir), c_float(sigma),
                                      stream_ptr()), "vx_ddim_step_eta")


def ddim_step_frames(latents, acc, frames, sqrt_a, sqrt_1ma, sqrt_aprev, sqrt_1maprev):
    """ddim_step on the frames listed in ``frames`` (int32 device tensor) of latents bf16 (n,4,L,h,w) / acc fp32
    (n,4,L,h*w); those acc entries are zeroed in the same pass."""
    n, c, L = latents.shape[:3]
    hw = latents[0, 0, 0].numel()
    if not (latents.dtype == BF16 and acc.dtype == torch.float32 and frames.dtype == torch.int32):
        raise ValueError(f"ddim_step_frames: latents bf16 / acc fp32 / frames int32, got {latents.dtype} / {acc.dtype} / "
                         f"{frames.dtype}")
    if not (latents.is_contiguous() and acc.is_contiguous() and frames.is_contiguous() and acc.numel() == latents.numel()
            and acc.shape[:3] == latents.shape[:3] and frames.dim() == 1 and 1 <= frames.numel() <= L):
        raise ValueError(f"ddim_step_frames: latents {tuple(latents.shape)} and acc {tuple(acc.shape)} must be contiguous "
                         f"(n,4,L,...) of equal size, frames a 1-D list of at most L indices, got {tuple(frames.shape)}")
    check(_ffi.lib().vx_ddim_step_frames(ptr(latents), ptr(acc), c_int(n * c), c_int(L), c_int(hw), ptr(frames),
                                         c_int(frames.numel()), c_float(sqrt_a), c_float(sqrt_1ma), c_float(sqrt_aprev),
                                         c_float(sqrt_1maprev), stream_ptr()), "vx_ddim_step_frames")


def _dpm_args(alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order):
    if order not in (1, 2):
        raise ValueError(f"dpmpp_step: order must be 1 or 2, got {order!r}")
    return (c_float(alpha_s), c_float(sigma_s), c_float(ratio), c_float(c0), c_float(inv_r0), c_float(c0h), c_int(order))


def dpmpp_step(latents, acc, x0_prev, alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order):
    """DPM-Solver++ step on all elements of latents bf16 (n,4,L,...): acc fp32 is the averaged model output, x0_prev bf16
    the previous step's x0 prediction (read at order 2), overwritten with this step's; scalars from
    ``scheduler.dpm_coefficients``."""
    if not (latents.dtype == BF16 and acc.dtype == torch.float32 and x0_prev.dtype == BF16):
        raise ValueError(f"dpmpp_step: latents bf16 / acc fp32 / x0_prev bf16, got {latents.dtype} / {acc.dtype} / "
                         f"{x0_prev.dtype}")
    if not (latents.is_contiguous() and acc.is_contiguous() and x0_prev.is_contiguous()
            and acc.numel() == latents.numel() == x0_prev.numel() and latents.device == acc.device == x0_prev.device):
        raise ValueError(f"dpmpp_step: latents {tuple(latents.shape)}, acc {tuple(acc.shape)} and x0_prev "
                         f"{tuple(x0_prev.shape)} must be contiguous tensors of equal size on one device")
    check(_ffi.lib().vx_dpmpp_step(ptr(latents), ptr(acc), ptr(x0_prev), c_ll(latents.numel()),
                                   *_dpm_args(alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order), stream_ptr()),
          "vx_dpmpp_step")


def dpmpp_step_frames(latents, acc, x0_prev, frames, alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order):
    """dpmpp_step on the frames listed in ``frames`` (int32 device tensor) of latents bf16 (n,4,L,h,w) / acc fp32 /
    x0_prev bf16 (n,4,L,h*w); those acc entries are zeroed in the same pass."""
    n, c, L = latents.shape[:3]
    hw = latents[0, 0, 0].numel()
    if not (latents.dtype == BF16 and acc.dtype == torch.float32 and x0_prev.dtype == BF16
            and frames.dtype == torch.int32):
        raise ValueError(f"dpmpp_step_frames: latents bf16 / acc fp32 / x0_prev bf16 / frames int32, got {latents.dtype} "
                         f"/ {acc.dtype} / {x0_prev.dtype} / {frames.dtype}")
    if not (latents.is_contiguous() and acc.is_contiguous() and x0_prev.is_contiguous() and frames.is_contiguous()
            and acc.numel() == latents.numel() == x0_prev.numel() and acc.shape[:3] == latents.shape[:3]
            and x0_prev.shape[:3] == latents.shape[:3] and frames.dim() == 1 and 1 <= frames.numel() <= L):
        raise ValueError(f"dpmpp_step_frames: latents {tuple(latents.shape)}, acc {tuple(acc.shape)} and x0_prev "
                         f"{tuple(x0_prev.shape)} must be contiguous (n,4,L,...) of equal size, frames a 1-D list of at "
                         f"most L indices, got {tuple(frames.shape)}")
    check(_ffi.lib().vx_dpmpp_step_frames(ptr(latents), ptr(acc), ptr(x0_prev), c_int(n * c), c_int(L), c_int(hw),
                                          ptr(frames), c_int(frames.numel()),
                                          *_dpm_args(alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order), stream_ptr()),
          "vx_dpmpp_step_frames")


def softmax_rows(x, out=None):
    """Row softmax of fp32 scores [rows, n] -> bf16 probabilities."""
    _chk_vectors("softmax_rows", 4, x, out)
    assert x.dtype == torch.float32 and x.stride(1) == 1
    rows, n = x.shape
    if out is None:
        out = torch.empty((rows, n), device=x.device, dtype=BF16)
    check(_ffi.lib().vx_softmax_rows(ptr(x), c_ll(x.stride(0)), c_ll(rows), c_int(n), ptr(out), c_ll(out.stride(0)),
                                     stream_ptr()), "vx_softmax_rows")
    return out


def pack_conv_out(w, bias, pad_to=32):
    """(Cout<=8, Cin, 3, 3) conv weight -> zero-padded [pad_to, 9*Cin] bf16 + fp32 bias[pad_to] for the wgmma conv."""
    co = w.shape[0]
    wp = torch.zeros((pad_to,) + tuple(w.shape[1:]), device=w.device, dtype=BF16)
    wp[:co] = w.to(BF16)
    bp = torch.zeros(pad_to, device=w.device, dtype=torch.float32)
    bp[:co] = bias.float()
    return pack_conv3x3_weight(wp), bp


def conv_out_tc(x, NB, H, W, w_packed, b_packed, out, post=False):
    """conv_out on the tensor-core conv kernel: x NHWC [NB*H*W, C]; out planar (n, co, h, w) bf16/fp32."""
    tmp = conv3x3(x.view(NB, H, W, -1), w_packed, b_packed)
    assert out.stride(3) == 1 and out.stride(2) == W
    check(_ffi.lib().vx_extract_planar(ptr(tmp), c_ll(tmp.stride(0)), c_int(NB), c_int(H * W), c_int(out.shape[1]),
                                       ptr(out), c_ll(out.stride(0)), c_ll(out.stride(1)),
                                       c_int(int(out.dtype == torch.float32)), c_int(int(post)), stream_ptr()),
          "vx_extract_planar")
    return out


def median3d_u8(video, want_filtered=False):
    """video (C,T,H,W) fp32 on the device -> uint8 frames (T,H,W,C) [, filtered (C,T,H,W) fp32]: the reference's
    ``median_filter_3d(kernel_size=3)`` + ``(v * 255).astype(uint8)`` (pipelines/utils.py:46-63,70-73)."""
    assert video.dtype == torch.float32 and video.is_contiguous() and video.dim() == 4
    C, T, H, W = video.shape
    frames = torch.empty((T, H, W, C), device=video.device, dtype=torch.uint8)
    filt = torch.empty_like(video) if want_filtered else None
    check(_ffi.lib().vx_median3d_u8(ptr(video), c_int(C), c_int(T), c_int(H), c_int(W), ptr(filt), ptr(frames),
                                    stream_ptr()), "vx_median3d_u8")
    return (frames, filt) if want_filtered else frames


def median3d_range_u8(buf, buf_start, own_start, own_count, video_length, out=None):
    """median3d_u8 of frames [own_start, own_start + own_count) of a ``video_length``-frame video from buf (C,k,H,W) fp32,
    which holds frames [buf_start, buf_start + k) including one neighbour on each side of the owned run (fewer at the
    video's ends) -> uint8 (own_count,H,W,C), bit-identical to those frames of median3d_u8 on the whole video."""
    if not (buf.dtype == torch.float32 and buf.is_contiguous() and buf.dim() == 4):
        raise ValueError(f"median3d_range_u8: buf must be a contiguous (C,k,H,W) fp32 tensor, got {buf.dtype} "
                         f"{tuple(buf.shape)}")
    C, k, H, W = buf.shape
    if out is None:
        out = torch.empty((own_count, H, W, C), device=buf.device, dtype=torch.uint8)
    if out.shape != (own_count, H, W, C) or out.dtype != torch.uint8 or not out.is_contiguous():
        raise ValueError(f"median3d_range_u8: out must be a contiguous uint8 {(own_count, H, W, C)}, got {tuple(out.shape)}")
    check(_ffi.lib().vx_median3d_range_u8(ptr(buf), c_int(C), c_int(k), c_int(buf_start), c_int(own_start),
                                          c_int(own_count), c_int(video_length), c_int(H), c_int(W), ptr(out),
                                          stream_ptr()), "vx_median3d_range_u8")
    return out


def im2col3x3(x, NB, H, W, stride=1, silu=False, out=None, pad_lo=1):
    """x [NB*H*W, C] NHWC bf16 -> [NB*Ho*Wo, 9*C] (pad 1; pad_lo=0: pad (0,1,0,1) at stride 2), optionally SiLU(x) while
    gathering."""
    _chk_bf16(x, out)
    C = x.shape[1]
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty((NB * Ho * Wo, 9 * C), device=x.device, dtype=BF16)
    # the kernel takes no leading dimensions: rows of x are C apart and rows of out 9 C apart
    if not x.is_contiguous() or x.shape[0] != NB * H * W or not out.is_contiguous() or out.shape != (NB * Ho * Wo, 9 * C):
        raise ValueError(f"im2col3x3: x must be a contiguous [{NB * H * W}, C] and out a contiguous [{NB * Ho * Wo}, {9 * C}] "
                         f"tensor, got x {tuple(x.shape)} strides {x.stride()}, out {tuple(out.shape)} strides {out.stride()}")
    check(_ffi.lib().vx_im2col3x3(ptr(x), c_int(NB), c_int(H), c_int(W), c_int(C), c_int(stride), c_int(int(silu)),
                                  c_int(pad_lo), ptr(out), stream_ptr()), "vx_im2col3x3")
    return out
