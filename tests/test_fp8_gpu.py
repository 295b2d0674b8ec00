"""FP8 mode on the H100: the LayerNorm -> e4m3 kernel, the e4m3 GEMM and the UNet forward with enable_fp8_linear().

LayerNorm -> e4m3 (ops.layernorm_fp8) against an fp64 LayerNorm of the same bf16 input: every code times its row scale is
within half an e4m3 step of the fp64 value (2^-4 relative for normal codes, half the subnormal step 2^-10 scale below
2^-6 scale), plus the fp32 LayerNorm's own error; the row scale equals amax / 448 of the fp64 row to fp32 precision, up to
the same LayerNorm error.  The fp32 LayerNorm error of an element is bounded by 2^-18 rstd |gamma| max|x_row| (the fp32
mean, 1 / C is not exact, is off by a few 2^-24 max|x_row|, and x - mean carries that, amplified by rstd: near-constant
rows) plus 2^-20 |y| (rstd, the products, + beta, + pe).

e4m3 GEMM (ops.gemm_fp8) against an fp64 reference of the dequantised operands A = codes_a * a_scale, W = codes_w *
w_scale, element by element, in the style of tests/test_gemm_bounds_gpu.py:

    |out - ref| <= 2^-8 |ref| + 2^-12 chain_abs + 2^-22 prod_abs + 2^-20 ref_abs
    chain_abs = sum_k |a_k w_k| (S - floor(k / 32)),    S = ceil(K / 32)

* 2^-8 |ref|: the rounding of the output to bf16.
* 2^-12 chain_abs: the accumulator this ASSUMES.  The kernel keeps one accumulator over the whole K and chains S
  m64nNk32 e4m3 MMAs into it.  The products of two e4m3 codes (4 significant bits each) are exact, but the tensor cores
  do not add them in fp32.  The model: every k32 MMA aligns its addends (incoming accumulator + 32 products) to the
  largest exponent e among them and keeps 14 significant bits, truncating; the error is below 2^(e + 1 - 14), i.e.
  2^-12 of the largest magnitude involved (>= 2^e), which is at most the running sum sum_{k < 32 (j + 1)} |a_k w_k|
  after step j.  Summed over the S steps that is chain_abs.  An fp32 accumulator bound (K 2^-22 prod_abs) is missed by
  up to x6 at every covered shape, which is why the fp32 model is not the one stated; on the ``cancel`` cases the kernel
  reaches 0.65 of this bound at K = 64 (2^-12 prod_abs), less at longer K.
* 2^-22 prod_abs: the two fp32 multiplications by a_scale[m] * w_scale[n].
* 2^-20 ref_abs: bias / scale / residual in fp32.
GEGLU propagates the same accumulation term of the value and gate columns as geglu_ref64 does.  The ``cancel`` cases add
a residual of -bf16(A W^T): the output is a small difference of large terms, so the accumulation error is not hidden under
the output rounding.

``test_fp8_bound_rejects_injected_faults`` (no GPU) runs a torch model of the kernel's arithmetic with a wrong row scale,
a wrong column scale, the scales applied twice, a K block dropped and (at K = 320) a bf16 accumulator (8 significant bits,
rounded after every k32 step) through the same check.  Over a long K the chain term, linear in the number of steps, grows
faster than a rounding accumulator's error, so the bf16 accumulator is only told apart at short K.

UNet forward: e(GPU fp8) <= 1.1 (e(emulated fp8) + e(GPU bf16)), every e the relative L2 error against the fp32 oracle on
the same bf16-rounded weights; disable_fp8_linear() restores bit-identical bf16 outputs; with FP8 on, a two-sample
forward equals the one-sample forwards bit for bit."""
import math
import os

import pytest
import torch

import fp8_emulation as E
from test_gemm_bounds_gpu import _SENTINEL, bound_check, linear_ref64
from test_unet_gpu import _rel, build_product

E4M3 = torch.float8_e4m3fn
_NAN8 = 0x7F                   # an e4m3 NaN code: cells around an e4m3 operand hold it


# ---------------------------------------------------------------------------------------------------------- references
def chain_abs64(A, W):
    """sum_k |a_k w_k| (S - floor(k / 32)), S = ceil(K / 32): the running sums a chain of k32 MMAs passes through"""
    K = A.shape[1]
    wts = (math.ceil(K / 32) - torch.arange(K, device=A.device) // 32).double()
    return (A.abs() * wts) @ W.abs().t()


def _gelu64(G):
    return 0.5 * G * (1 + torch.erf(G / math.sqrt(2)))


def fp8_ref64(a8, a_scale, w8, w_scale, bias=None, residual=None, geglu=False):
    """(ref, bound without the output rounding) of the e4m3 GEMM; w8 / w_scale / bias unpacked for GEGLU."""
    A = a8.double() * a_scale.double()[:, None]
    W = w8.double() * w_scale.double()[:, None]
    if not geglu:
        ref, ref_abs, prod_abs = linear_ref64(A, W, bias, residual=residual)
        return ref, 2.0 ** -12 * chain_abs64(A, W) + 2.0 ** -22 * prod_abs + 2.0 ** -20 * ref_abs
    # GEGLU: the error propagation of geglu_ref64 (tests/test_gemm_bounds_gpu.py) with this accumulation term
    inner = W.shape[0] // 2
    V, _, Pv = linear_ref64(A, W[:inner], bias[:inner])
    G, _, Pg = linear_ref64(A, W[inner:], bias[inner:])
    dV = 2.0 ** -12 * chain_abs64(A, W[:inner]) + 2.0 ** -22 * (2 * Pv + bias[:inner].double().abs())
    dG = 2.0 ** -12 * chain_abs64(A, W[inner:]) + 2.0 ** -22 * (2 * Pg + bias[inner:].double().abs())
    gl = _gelu64(G)
    dgelu = (0.5 * (1 + torch.erf(G / math.sqrt(2))) + G * torch.exp(-0.5 * G * G) / math.sqrt(2 * math.pi)).abs()
    d1 = torch.clamp(dgelu + 0.8 * dG, max=1.13)
    e_gelu = G.abs() * (2.0 ** -22 + 2.0 ** -18 * torch.erfc(G.abs() / math.sqrt(2))) + 2.0 ** -21 * gl.abs()
    return V * gl, gl.abs() * dV + V.abs() * (d1 * dG + e_gelu) + dV * (1.13 * dG + e_gelu) + 2.0 ** -22 * (V * gl).abs()


def quantize_rows(x):
    codes, scale = E.quantize_rows(x)
    return codes, scale.reshape(-1)


def fp8_operands(g, M, K, N, dev="cpu"):
    """e4m3 A [M, K] / W [N, K] with per-row scales; rows over four decades (the scales differ from row to row), and the
    128-element K blocks (one ring stage) of A scaled alternately by 4 and 1/4 so that every block carries weight."""
    rn = lambda *s: torch.randn(*s, generator=g)
    blk = torch.where((torch.arange(K) // 128) % 2 == 0, 4.0, 0.25)
    A = rn(M, K) * torch.logspace(-2, 2, M)[torch.randperm(M, generator=g)].view(-1, 1) * blk
    W = rn(N, K) / math.sqrt(K) * torch.logspace(-1, 1, N)[torch.randperm(N, generator=g)].view(-1, 1)
    a8, sa = quantize_rows(A)
    w8, sw = quantize_rows(W)
    return a8.to(dev), sa.to(dev), w8.to(dev), sw.to(dev)


def emulate_fp8_gemm(a8, a_scale, w8, w_scale, bias=None, fault=None):
    """torch model of the kernel: fp32 sum of code products, * a_scale[m] * w_scale[n], + bias, rounded to bf16."""
    A, W = a8.float(), w8.float()
    sa, sw = a_scale.clone(), w_scale.clone()
    if fault == "k_block_dropped":
        A[:, :128] = 0
    if fault == "row_scale":
        sa = sa.roll(1)
    if fault == "col_scale":
        sw = sw.roll(1)
    if fault == "bf16_accumulator":
        acc = torch.zeros(A.shape[0], W.shape[0])
        for k0 in range(0, A.shape[1], 32):
            acc = (acc + A[:, k0:k0 + 32] @ W[:, k0:k0 + 32].t()).bfloat16().float()
    else:
        acc = A @ W.t()
    out = acc * (sa[:, None] * sw[None, :])
    if fault == "scale_twice":
        out = out * (sa[:, None] * sw[None, :])
    if bias is not None:
        out = out + bias
    return out.bfloat16()


FAULTS = ("row_scale", "col_scale", "scale_twice", "k_block_dropped", "bf16_accumulator")


@pytest.mark.parametrize("K", [320, 1280])
def test_fp8_bound_rejects_injected_faults(K):
    g = torch.Generator().manual_seed(5)
    a8, sa, w8, sw = fp8_operands(g, 200, K, 96)
    bias = torch.randn(96, generator=g)
    ref, bnd = fp8_ref64(a8, sa, w8, sw, bias)
    worst, _, where = bound_check(emulate_fp8_gemm(a8, sa, w8, sw, bias), ref, bnd)
    assert worst <= 1, where
    for fault in FAULTS:
        if fault == "bf16_accumulator" and K > 320:
            continue
        worst, _, where = bound_check(emulate_fp8_gemm(a8, sa, w8, sw, bias, fault), ref, bnd)
        print(f"K={K} {fault}: {where}")
        assert worst > 1, (fault, where)


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture
def schedule():
    """schedule(pp): VX_GEMM_PP = pp for the library (0 cooperative, 1 ping-pong wherever the kernel has it)."""
    from vexpress_b200 import _ffi
    before = os.environ.get("VX_GEMM_PP")

    def switch(pp):
        os.environ["VX_GEMM_PP"] = str(pp)
        _ffi.lib().vx_gemm_reload_env()

    yield switch
    if before is None:
        os.environ.pop("VX_GEMM_PP", None)
    else:
        os.environ["VX_GEMM_PP"] = before
    _ffi.lib().vx_gemm_reload_env()


def _bordered(rows, cols, dtype):
    """[rows, cols] interior view of a sentinel-filled buffer (16 columns more on either side, rows above and below): the
    e4m3 rows start 16-byte aligned, as TMA needs."""
    if dtype == E4M3:
        buf = torch.full((rows + 8, cols + 32), _NAN8, dtype=torch.uint8, device="cuda").view(E4M3)
    elif dtype == torch.float32:
        buf = torch.full((rows + 8, cols + 32), float("nan"), dtype=torch.float32, device="cuda")
    else:
        buf = torch.full((rows + 8, cols + 32), _SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return buf, buf[3:3 + rows, 16:16 + cols]


def _border_intact(buf, rows, cols):
    b = buf.view(torch.uint8) if buf.dtype == E4M3 else buf
    mask = torch.ones(b.shape, dtype=torch.bool, device=b.device)
    mask[3:3 + rows, 16:16 + cols] = False
    outside = b[mask]
    if buf.dtype == E4M3:
        return bool((outside == _NAN8).all())
    if buf.dtype == torch.float32:
        return bool(torch.isnan(outside).all())
    return bool((outside.view(torch.int16) == _SENTINEL).all())


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 320, 640, 1280])
@pytest.mark.parametrize("pe", [False, True])
def test_layernorm_fp8(ops, C, pe):
    g = torch.Generator().manual_seed(C + pe)
    rows_per_frame, frames = 37, 5                      # frame edges inside every kernel's row groups
    rows = rows_per_frame * frames * 2 + 11
    x = torch.randn(rows, C, generator=g) * torch.logspace(-1, 1, rows).view(-1, 1) + torch.randn(rows, 1, generator=g)
    x[7] = 3.0                                          # constant row: LayerNorm gives beta (+ pe)
    gamma, beta = 1 + 0.3 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    pe_t = torch.randn(frames, C, generator=g) if pe else None
    xb = x.bfloat16()
    xbuf, xv = _bordered(rows, C, torch.bfloat16)
    xv.copy_(xb.cuda())
    obuf, ov = _bordered(rows, C, E4M3)
    sbuf = torch.full((rows + 4,), float("nan"), device="cuda")
    dev = lambda t: None if t is None else t.float().cuda().contiguous()
    codes, scale = ops.layernorm_fp8(xv, dev(gamma), dev(beta), pe=dev(pe_t), rows_per_frame=rows_per_frame if pe else 0,
                                     out=ov, row_scale=sbuf[:rows])
    torch.cuda.synchronize()
    assert _border_intact(obuf, rows, C) and torch.isnan(sbuf[rows:]).all()
    # fp64 LayerNorm of the bf16 input
    xd = xb.double()
    mu = xd.mean(1, keepdim=True)
    var = ((xd - mu) ** 2).mean(1, keepdim=True)
    y = (xd - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()
    if pe:
        y = y + pe_t.double()[(torch.arange(rows) // rows_per_frame) % frames]
    e_ln = (2.0 ** -18 * torch.rsqrt(var + 1e-5) * gamma.double().abs() * xd.abs().amax(1, keepdim=True)
            + 2.0 ** -20 * y.abs())
    amax = y.abs().amax(1)
    s_ref = torch.where(amax > 0, amax / 448, torch.ones_like(amax))
    s = scale.double().cpu()
    s_err = (s - s_ref).abs() / (e_ln.amax(1) / 448 + 2.0 ** -22 * s_ref)
    assert (s_err <= 1).all(), s_err.max()
    deq = codes.cpu().double() * s[:, None]
    assert not torch.isnan(deq).any()
    half_step = torch.maximum(y.abs() * 2.0 ** -4, 2.0 ** -10 * s[:, None])
    err = (deq - y).abs()
    bound = half_step * (1 + 2.0 ** -20) + 2 * e_ln
    ratio = (err / bound).max().item()
    print(f"C={C} pe={pe}: worst |code * scale - LayerNorm| / bound = {ratio:.3f}")
    assert ratio <= 1


CASES = [  # (K, N, geglu, cancel): the covered shapes of a forward (K = C, N = 3C / C / 8C GEGLU), the reduced widths,
    # and outputs that cancel to near zero
    *[(C, n, gg, False) for C in (320, 640, 1280) for n, gg in ((3 * C, False), (C, False), (8 * C, True))],
    (64, 192, False, False), (64, 64, False, False), (64, 512, True, False), (128, 384, False, False),
    (256, 2048, True, False), (96, 96, False, False),
    *[(K, 256, False, True) for K in (64, 320, 640, 1280)],
]


@pytest.mark.gpu
@pytest.mark.parametrize("pp", [0, 1])
@pytest.mark.parametrize("K,N,geglu,cancel", CASES)
def test_gemm_fp8_bound(ops, schedule, K, N, geglu, cancel, pp):
    schedule(pp)
    g = torch.Generator().manual_seed(K * 7 + N + geglu)
    M = 1000 + K % 77                                   # not a multiple of the 128-row tile
    a8, sa, w8, sw = fp8_operands(g, M, K, N)
    bias = torch.randn(N, generator=g) if (geglu or N != 3 * K) else None
    residual = None if geglu or bias is None else torch.randn(M, N, generator=g).bfloat16()
    if cancel:   # -bf16(A W^T + b): the output is what the accumulation and rounding leave over
        A64, W64 = a8.double() * sa.double()[:, None], w8.double() * sw.double()[:, None]
        residual = (-(A64 @ W64.t() + bias.double())).bfloat16()
    ref, bnd = fp8_ref64(a8.cuda(), sa.cuda(), w8.cuda(), sw.cuda(), None if bias is None else bias.cuda(),
                         None if residual is None else residual.cuda(), geglu)
    abuf, av = _bordered(M, K, E4M3)
    av.copy_(a8.cuda())
    dev = lambda t: None if t is None else t.float().cuda().contiguous()
    bn = 0
    if geglu:
        bn = 128 if pp else 256                         # ping-pong needs a packing at one of its widths
        wp, bp, bn = ops.pack_geglu(w8.view(torch.uint8), bias, bn)
        swp, _, _ = ops.pack_geglu(sw.view(-1, 1), None, bn)
        wbuf, wv = _bordered(N, K, E4M3)
        wv.copy_(wp.view(E4M3).cuda())
        sw_d, b_d = dev(swp.view(-1)), dev(bp)
    else:
        wbuf, wv = _bordered(N, K, E4M3)
        wv.copy_(w8.cuda())
        sw_d, b_d = dev(sw), dev(bias)
    out_n = N // 2 if geglu else N
    obuf, ov = _bordered(M, out_n, torch.bfloat16)
    rbuf, rv = (None, None) if residual is None else _bordered(M, N, torch.bfloat16)
    if rv is not None:
        rv.copy_(residual.cuda())
    ops.gemm_fp8(av, dev(sa), wv, sw_d, b_d, residual=rv, out=ov, geglu=geglu, block_n=bn)
    torch.cuda.synchronize()
    assert _border_intact(obuf, M, out_n)
    worst, rel, where = bound_check(ov, ref, bnd, residual=residual.cuda() if residual is not None else None)
    print(f"K={K} N={N} geglu={geglu} cancel={cancel} pp={pp}: {where}, rel {rel:.2e}")
    assert worst <= 1, where
    assert rel < 5e-3


# ------------------------------------------------------------------------------------------------------------ the UNet
def _unet_case(cfg, sd, f, h, seed):
    from oracle import vx_oracle as O
    lat, kps, audio, banks = O.synth_inputs(cfg, f, h, h, True, seed)
    model, reader = build_product(cfg, sd, [b[1:] for b in banks], 0.95, 3.0)
    x = lat.repeat(2, 1, 1, 1, 1)
    enc = audio.reshape(-1, 5, cfg["cross_attention_dim"])
    return model, reader, x, enc, kps, banks


def _run(model, x, enc, kps):
    with torch.no_grad():
        out = model(x.bfloat16().cuda(), 499, encoder_hidden_states=enc.bfloat16().cuda(), kps_features=kps.bfloat16().cuda(),
                    return_dict=False)[0]
    torch.cuda.synchronize()
    return out


def _check_unet(cfg, sd, f, h, seed):
    from oracle import vx_oracle as O
    model, reader, x, enc, kps, banks = _unet_case(cfg, sd, f, h, seed)
    out16 = _run(model, x, enc, kps)
    model.enable_fp8_linear()
    out8 = _run(model, x, enc, kps)
    model.disable_fp8_linear()
    out16b = _run(model, x, enc, kps)
    reader.clear()
    assert torch.equal(out16b, out16)
    assert not torch.equal(out8, out16)
    r = lambda t: t.bfloat16().float()
    args = ({k: r(v) for k, v in sd.items()}, cfg, r(x), 499, r(enc), r(kps), [r(b) for b in banks], 0.95, 3.0)
    with torch.no_grad():
        ref = O.unet_forward(*args)
        emu = E.unet_forward_fp8(*args)
    e8, e16, e_emu = _rel(out8.float().cpu(), ref), _rel(out16.float().cpu(), ref), _rel(emu, ref)
    print(f"vs fp32 oracle: GPU fp8 {e8:.4%}, emulated fp8 {e_emu:.4%}, GPU bf16 {e16:.4%}")
    assert e8 <= 1.1 * (e_emu + e16)


@pytest.mark.gpu
def test_unet_fp8_reduced_width(golden_dir):
    from oracle import vx_oracle as O
    g = torch.load(os.path.join(golden_dir, "unet_small.pt"), weights_only=False)
    cfg = g["cfg"]
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), g["seed_weights"])
    _check_unet(cfg, sd, g["f"], g["h"], g["seed_inputs"])


@pytest.mark.gpu
def test_unet_fp8_full_width_and_samples():
    """configs[0] shape (f = 4, 64x64 latents), full width, against the fp32 oracle on the CPU.  Then, with FP8 on, one
    forward of [u s0 | u s1 | c s0 | c s1] equals the two one-sample forwards with torch.equal."""
    from oracle import vx_oracle as O
    cfg = O.DEFAULT_CFG
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
    f, h = 4, 64
    _check_unet(cfg, sd, f, h, 42)
    lat, kps, audio, banks = O.synth_inputs(cfg, f, h, h, True, 42)
    model, reader = build_product(cfg, sd, [b[1:] for b in banks], 0.95, 3.0)
    model.enable_fp8_linear()
    eng = model.engine()
    assert eng.fp8
    lat2 = torch.randn(lat.shape, generator=torch.Generator().manual_seed(7))
    samples = [lat[0].transpose(0, 1).bfloat16().cuda(), lat2[0].transpose(0, 1).bfloat16().cuda()]
    kps_nhwc = kps.bfloat16().cuda().permute(0, 2, 3, 4, 1).reshape(2 * f * h * h, -1).contiguous()
    enc = audio.reshape(2, f, 5, cfg["cross_attention_dim"]).bfloat16().cuda()
    idx1 = torch.arange(2 * f, device="cuda", dtype=torch.int32)
    with torch.no_grad():
        one = [eng.forward_frames(torch.cat([x, x]), 499, enc.reshape(-1, 5, enc.shape[-1]), kps_nhwc, idx1, 2, f)
               for x in samples]
        frames = torch.cat(samples + samples)
        enc2 = enc.unsqueeze(1).expand(2, 2, f, 5, enc.shape[-1]).reshape(-1, 5, enc.shape[-1]).contiguous()
        idx2 = idx1.view(2, 1, f).expand(2, 2, f).reshape(-1).contiguous()
        two = eng.forward_frames(frames, 499, enc2, kps_nhwc, idx2, 2, f, n=2).view(2, 2, f, 4, h, h)
    torch.cuda.synchronize()
    reader.clear()
    for s in range(2):
        assert torch.equal(two[:, s], one[s].view(2, f, 4, h, h)), s


def test_enable_fp8_rejects_ln_fold(monkeypatch):
    from vexpress_b200.modules.unet_3d import _check_fp8_env
    for var in ("VX_LN_FOLD", "VX_LN_FUSE"):
        monkeypatch.setenv(var, "1")
        with pytest.raises(ValueError):
            _check_fp8_env()
        monkeypatch.delenv(var)
    _check_fp8_env()
