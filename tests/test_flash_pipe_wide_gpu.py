"""The pipelined flash-attention loop at hd 80 and 160 (one CTA per SM with two consumer warpgroups, or two CTAs per SM
with one) against the serial loop, bit for bit, on the edges the UNet's shapes do not reach: a masked key tail, a query
tile that runs into the next frame and past the last row, one consumer warpgroup over several steps, and, at hd 160,
fewer ring stages than steps (GPU)."""
import pytest
import torch

from test_zz_flash_pipeline_gpu import _inputs, ops, serial_loop  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

# (B, N, heads, hd, kv_div, Nk)
_SHAPES = [(3, 384, 8, 80, 3, 336),     # Nk = 5 x 64 + 16: the key tail is masked under two consumers
           (2, 192, 8, 80, 1, 592),     # Nq not a multiple of 128; Nk = 9 x 64 + 16
           (2, 80, 8, 160, 1, 80),      # tiles past the last row, masked tail
           (4, 64, 8, 80, 2, 400),      # one consumer warpgroup, seven steps, masked tail
           (2, 64, 4, 160, 1, 1040),    # one consumer warpgroup, a 2-stage ring over 17 steps
           (2, 512, 8, 160, 2, 1024)]   # two consumers, a 4-stage ring over 16 steps


@pytest.mark.parametrize("B,N,heads,hd,kv_div,Nk,family",
                         [pytest.param(*s, f, id="-".join(map(str, s)) + "-" + f)
                          for f in ("flat", "peaked", "tail") for s in _SHAPES])
def test_wide_pipelined_loop_equals_serial_loop(ops, serial_loop, B, N, heads, hd, kv_div, Nk, family):  # noqa: F811
    q, k, v = _inputs(B, N, heads, hd, kv_div, Nk, family)
    serial_loop(True)
    ref = ops.flash_attention(q, k, v, heads, N, Nk, kv_div)
    serial_loop(False)
    out = ops.flash_attention(q, k, v, heads, N, Nk, kv_div)
    torch.cuda.synchronize()
    assert not torch.isnan(out.float()).any()
    assert torch.equal(out, ref), f"max abs diff {(out.float() - ref.float()).abs().max().item():.3e}"
