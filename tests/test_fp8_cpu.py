"""FP8 mode without a GPU: the weight quantiser reproduces its documented formula bit for bit (fused q|k|v and GEGLU packings
included), and the CPU emulation of the scheme gives the documented error on the reduced-width golden UNet."""
import os

import pytest
import torch

from vexpress_b200 import ops

import fp8_emulation as E


def _codes_equal(a, b):
    return a.dtype == b.dtype == torch.float8_e4m3fn and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _weight(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * torch.logspace(-3, 1, N).view(-1, 1)   # rows over four decades
    w[3] = 0.0                                                                  # all-zero output channel
    w[5, 7] = 300.0                                                             # one outlier dominates its row
    return w.bfloat16()


def test_torch_cast_does_not_saturate():
    # why quantize_fp8_weight clamps before the cast
    x = torch.tensor([449.0, 464.0, 500.0])
    y = x.to(torch.float8_e4m3fn).float()
    assert y[0] == 448 and y[1] == 448 and torch.isnan(y[2])


def test_quantize_fp8_weight_formula():
    w = _weight(96, 320, 0)
    codes, scale = ops.quantize_fp8_weight(w)
    wf = w.float()
    amax = wf.abs().amax(1)
    s = torch.where(amax > 0, amax / 448, torch.ones_like(amax))
    assert scale.dtype == torch.float32 and torch.equal(scale, s)
    assert scale[3] == 1.0
    assert _codes_equal(codes, (wf / s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn))
    assert not torch.isnan(codes.float()).any()
    assert codes.float().abs().amax(1)[torch.arange(96) != 3].eq(448).all()   # every non-zero row reaches the e4m3 maximum
    # codes * scale is within half an e4m3 step of w (2^-4 relative, or half the subnormal step 2^-10 scale)
    err = (codes.float() * scale[:, None] - wf).abs()
    assert (err <= torch.maximum(wf.abs() * 2.0 ** -4, 2.0 ** -10 * scale[:, None]) * (1 + 1e-6)).all()


def test_quantize_fp8_weight_fused_qkv_and_geglu():
    C = 128
    q, k, v = (_weight(C, C, s) for s in (1, 2, 3))
    cq, sq = ops.quantize_fp8_weight(torch.cat([q, k, v], 0))
    parts = [ops.quantize_fp8_weight(t) for t in (q, k, v)]
    assert _codes_equal(cq, torch.cat([p[0] for p in parts], 0))
    assert torch.equal(sq, torch.cat([p[1] for p in parts], 0))
    # GEGLU: codes and scales of the packed weight follow pack_geglu's per-tile (value | gate) interleave
    w = _weight(8 * C, C, 4)
    b = torch.randn(8 * C)
    wp, bp, bn = ops.pack_geglu(w, b)
    cg, sg = ops.quantize_fp8_weight(wp)
    c0, s0 = ops.quantize_fp8_weight(w)
    cpk, _, _ = ops.pack_geglu(c0.view(torch.uint8), None, bn)
    spk, _, _ = ops.pack_geglu(s0.view(-1, 1), None, bn)
    assert torch.equal(cg.view(torch.uint8), cpk) and torch.equal(sg, spk.view(-1))


def test_emulation_error_on_golden_unet(golden_dir):
    """Relative L2 error of the noise prediction against fp32 with the covered Linears' operands rounded to bf16 and to
    e4m3 (per-row / per-channel scales): 0.51 % and 7.5 % on the reduced-width golden UNet, t = 499."""
    from oracle import vx_oracle as O
    g = torch.load(os.path.join(golden_dir, "unet_small.pt"), weights_only=False)
    cfg = g["cfg"]
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), g["seed_weights"])
    lat, kps, audio, banks = O.synth_inputs(cfg, g["f"], g["h"], g["h"], True, g["seed_inputs"])
    x = lat.repeat(2, 1, 1, 1, 1)
    enc = audio.reshape(-1, 5, cfg["cross_attention_dim"])
    args = (sd, cfg, x, 499, enc, kps, banks, g["ref_w"], g["audio_w"])
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    with torch.no_grad():
        ref = O.unet_forward(*args)
        e8 = rel(E.unet_forward_fp8(*args), ref)
        with E.covered_linears(E.bf16_round, E.bf16_round) as hits:
            e16 = rel(O.unet_forward(*args), ref)
    # 16 spatial blocks x (q, k, v, attn1_5.to_q, attn2.to_q, ff) + 21 motion modules x (2 x (q, k, v) + ff)
    assert hits == E.covered_keys(sd) and len(hits) == 16 * 6 + 21 * 7
    print(f"covered Linears in e4m3: {e8:.4%}, in bf16: {e16:.4%}")
    assert e8 == pytest.approx(0.075, abs=5e-4)
    assert e16 == pytest.approx(0.0051, abs=5e-5)
