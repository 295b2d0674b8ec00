"""CPU statement of the FP8 mode (UNet3DConditionModel.enable_fp8_linear) on top of the fp32 oracle.

The covered Linears are the ones that read a LayerNorm output: attn1.to_q / to_k / to_v, attn1_5.to_q, attn2.to_q and
ff.net.0.proj of the spatial transformer blocks, attention_blocks.{0,1}.to_q / to_k / to_v and ff.net.0.proj of the motion
modules.  Under `unet_forward_fp8` each of them quantises its input to e4m3 with one scale per row (amax / 448) and its
weight with one scale per output channel, and multiplies the dequantised values in fp32.  Every other operation is the
oracle's own.  The GPU path is checked against this.

The oracle itself stays the fp32 statement of the reference; the scheme is applied by routing the oracle's Linear helper
(`_lin`, which every Linear of `unet_forward` goes through) for the duration of one call, under a lock, and the call fails
unless every covered Linear weight of the state dict was used -- so a change in how the oracle reaches its Linears cannot
silently turn the emulation back into fp32."""
import contextlib
import re
import threading

import torch
import torch.nn.functional as F

from oracle import vx_oracle as O

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0
COVERED = re.compile(r"\.(attn1\.to_[qkv]|attn1_5\.to_q|attn2\.to_q|attention_blocks\.\d\.to_[qkv]|ff\.net\.0\.proj)$")


def quantize_rows(t):
    """(e4m3 codes, fp32 scales) of t along its last dimension: scale = amax / 448 (1 for an all-zero row),
    codes = clamp(t / scale, +-448) rounded to nearest even."""
    t = t.float()
    amax = t.abs().amax(dim=-1, keepdim=True)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    return (t / scale).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3), scale


def fake_quant_rows(t):
    codes, scale = quantize_rows(t)
    return codes.float() * scale


def bf16_round(t):
    return t.bfloat16().float()


_LOCK = threading.Lock()


def covered_keys(sd):
    """module paths of the covered Linears in a UNet state dict"""
    return {k[:-len(".weight")] for k in sd if k.endswith(".weight") and COVERED.search(k[:-len(".weight")])}


@contextlib.contextmanager
def covered_linears(act=fake_quant_rows, weight=fake_quant_rows):
    """Within the block, the oracle's covered Linears compute F.linear(act(x), weight(W), b) in fp32.  Yields the set of
    covered module paths that were called."""
    hits = set()
    with _LOCK:
        orig = O._lin

        def lin(sd, p, x):
            if COVERED.search(p):
                hits.add(p)
                return F.linear(act(x), weight(sd[p + ".weight"]), sd.get(p + ".bias"))
            return orig(sd, p, x)

        O._lin = lin
        try:
            yield hits
        finally:
            O._lin = orig


def unet_forward_fp8(sd, *args, **kw):
    """oracle.vx_oracle.unet_forward with the covered Linears on e4m3 operands (per-row / per-output-channel scales)."""
    with covered_linears() as hits:
        out = O.unet_forward(sd, *args, **kw)
    missed = covered_keys(sd) - hits
    if missed or not hits:
        raise RuntimeError(f"fp8 emulation: {len(missed)} covered Linears did not go through the oracle's _lin "
                           f"(e.g. {sorted(missed)[:3]}); the emulation would be fp32 there")
    return out
