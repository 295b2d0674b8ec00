"""Conditioning prologue on the H100 kernels (SURVEY.md 8(f) row f2): drop-ins for the reference's
``modules/v_kps_guider.py`` (VKpsGuider) and ``modules/audio_projection.py`` (AudioProjection), same constructor
arguments, ``state_dict`` layout and ``forward`` signatures.  Both run once per video and are composed from the
hot path's validated operators plus one gather kernel:

* VKpsGuider (8 narrow 3x3 convs with SiLU in between, 512^2 -> 64^2): ``conv_in`` kernel for the 3-channel input, then
  every conv as ``im2col3x3(SiLU(x))`` + tensor-core GEMM with the channel counts padded to multiples of 32 by zero
  weights (the implicit-GEMM conv needs C % 64 == 0);
* AudioProjection (4-layer perceiver resampler, 10 -> 5 tokens per frame): GEMMs, LayerNorm, the exact-softmax attention
  kernel for the 15-key attention, GELU through the GEGLU epilogue with a constant-one value half.

Checked on the GPU by tests/test_prologue_bounds_gpu.py (every kernel call of a forward against an fp64 reference
under an elementwise bound, the modules against the fp64 oracle at 512^2 / 768^2 and L up to 1000, the chunking and
batching invariants) and tests/test_zz_prologue_gpu.py (the reference-generated golden).  Oracle: oracle/vx_oracle.py
(kps_guider_forward, audio_projection_forward); golden: tests/golden/prologue_small.pt.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
from torch import nn

from .. import ops
from .unet_3d import BF16, _Node


def _tree(root: nn.Module, shapes: Dict[str, Tuple[int, ...]]):
    for key, shape in shapes.items():
        parts = key.split(".")
        node = root
        for name in parts[:-1]:
            child = node._modules.get(name)
            if child is None:
                child = _Node()
                node.add_module(name, child)
            node = child
        node.register_parameter(parts[-1], nn.Parameter(torch.empty(shape), requires_grad=False))


def _pad32(c: int) -> int:
    return (c + 31) // 32 * 32


class VKpsGuider(nn.Module):
    """reference modules/v_kps_guider.py:10-45 (inference.py:100: VKpsGuider(320, block_out_channels=(16, 32, 96, 256)))."""

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                 block_out_channels: Tuple[int, ...] = (16, 32, 64, 128)):
        super().__init__()
        if conditioning_channels > 4:
            raise ValueError("vexpress_b200.VKpsGuider: at most 4 conditioning channels")
        self.cfg = (conditioning_embedding_channels, conditioning_channels, tuple(block_out_channels))
        boc = tuple(block_out_channels)
        S: Dict[str, Tuple[int, ...]] = {"conv_in.weight": (boc[0], conditioning_channels, 3, 3), "conv_in.bias": (boc[0],)}
        for i in range(len(boc) - 1):
            S[f"blocks.{2 * i}.weight"] = (boc[i], boc[i], 3, 3)
            S[f"blocks.{2 * i}.bias"] = (boc[i],)
            S[f"blocks.{2 * i + 1}.weight"] = (boc[i + 1], boc[i], 3, 3)
            S[f"blocks.{2 * i + 1}.bias"] = (boc[i + 1],)
        S["conv_out.weight"] = (conditioning_embedding_channels, boc[-1], 3, 3)
        S["conv_out.bias"] = (conditioning_embedding_channels,)
        _tree(self, S)
        self._packed = None

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    def _apply(self, fn, *a, **k):
        self._packed = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._packed = None
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _pack(self):
        if self._packed is not None:
            return self._packed
        dev = self.device
        sd = {k: v.detach().to(device=dev, dtype=BF16) for k, v in self.state_dict().items()}   # model-dtype rounding
        w0, b0 = sd["conv_in.weight"].float(), sd["conv_in.bias"].float()
        c0 = _pad32(w0.shape[0])
        w0p = torch.zeros(c0, 4, 3, 3, device=dev)
        w0p[:w0.shape[0], :w0.shape[1]] = w0
        b0p = torch.zeros(c0, device=dev)
        b0p[:b0.shape[0]] = b0
        first = (w0p.reshape(c0, 36).t().contiguous(), b0p, c0)                 # conv_in kernel: fp32 [Cin*9, Cout]
        layers: List[tuple] = []
        cin_pad = c0
        names = [f"blocks.{i}" for i in range(2 * (len(self.cfg[2]) - 1))] + ["conv_out"]
        for i, n in enumerate(names):
            w, b = sd[n + ".weight"], sd[n + ".bias"].float()
            cout_pad = _pad32(w.shape[0])
            wp = torch.zeros(cout_pad, cin_pad, 3, 3, device=dev, dtype=BF16)
            wp[:w.shape[0], :w.shape[1]] = w
            bp = torch.zeros(cout_pad, device=dev)
            bp[:b.shape[0]] = b
            stride = 2 if (n.startswith("blocks.") and int(n.split(".")[1]) % 2 == 1) else 1
            layers.append((ops.pack_conv3x3_weight(wp), bp, stride))
            cin_pad = cout_pad
        self._packed = (first, layers)
        return self._packed

    @torch.no_grad()
    def forward(self, conditioning: torch.Tensor, frames_per_chunk: int = 8) -> torch.Tensor:
        """conditioning (b, c, t, H, W) -> (b, C_emb, t, H/8, W/8) bf16 (reference :35-45; every conv is per-frame)."""
        from .. import _ffi
        _ffi.require_sm90()
        b, c, t, H, W = conditioning.shape
        (w0, b0, c0), layers = self._pack()
        dev = self.device
        x = conditioning.to(device=dev, dtype=BF16).permute(0, 2, 1, 3, 4).reshape(b * t, c, H, W)
        outs = []
        for n0 in range(0, b * t, frames_per_chunk):
            xc = x[n0:n0 + frames_per_chunk]
            n = xc.shape[0]
            xp = torch.zeros(n, 4, H, W, device=dev, dtype=BF16)
            xp[:, :c] = xc
            a = ops.conv_in(xp, w0, b0, c0)                                     # [n*H*W, c0], no activation yet
            h, w = H, W
            for wk, bk, stride in layers:
                col = ops.im2col3x3(a, n, h, w, stride=stride, silu=True)       # SiLU of the previous conv, then gather
                a = ops.gemm(col, wk, bk)
                h, w = (h - 1) // stride + 1, (w - 1) // stride + 1
            outs.append(a[:, :self.cfg[0]].reshape(n, h, w, self.cfg[0]))
        y = torch.cat(outs, 0)                                                  # (b*t, h, w, C)
        return y.view(b, t, y.shape[1], y.shape[2], y.shape[3]).permute(0, 4, 1, 2, 3).contiguous()


class AudioProjection(nn.Module):
    """reference modules/audio_projection.py:88-150 (inference.py:116-126: dim = embedding_dim = output_dim = 768,
    depth 4, dim_head 64, heads 12, num_queries 5, max_seq_len 10)."""

    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024,
                 ff_mult=4, max_seq_len: int = 257, num_latents_mean_pooled: int = 0):
        super().__init__()
        if num_latents_mean_pooled != 0:
            raise ValueError("vexpress_b200.AudioProjection: mean-pooled latents are not used by V-Express")
        if num_queries + max_seq_len > 64 or dim_head % 2:
            raise ValueError("vexpress_b200.AudioProjection: attention over more than 64 tokens is not supported")
        self.cfg = dict(dim=dim, depth=depth, dim_head=dim_head, heads=heads, num_queries=num_queries,
                        embedding_dim=embedding_dim, output_dim=output_dim, ff_mult=ff_mult, max_seq_len=max_seq_len)
        inner = dim_head * heads
        S: Dict[str, Tuple[int, ...]] = {"pos_emb.weight": (max_seq_len, embedding_dim), "latents": (1, num_queries, dim),
                                         "proj_in.weight": (dim, embedding_dim), "proj_in.bias": (dim,),
                                         "proj_out.weight": (output_dim, dim), "proj_out.bias": (output_dim,),
                                         "norm_out.weight": (output_dim,), "norm_out.bias": (output_dim,)}
        for i in range(depth):
            a, f = f"layers.{i}.0", f"layers.{i}.1"
            for nrm in ("norm1", "norm2"):
                S[f"{a}.{nrm}.weight"] = (dim,)
                S[f"{a}.{nrm}.bias"] = (dim,)
            S[a + ".to_q.weight"] = (inner, dim)
            S[a + ".to_kv.weight"] = (2 * inner, dim)
            S[a + ".to_out.weight"] = (dim, inner)
            S[f + ".0.weight"] = (dim,)
            S[f + ".0.bias"] = (dim,)
            S[f + ".1.weight"] = (ff_mult * dim, dim)
            S[f + ".3.weight"] = (dim, ff_mult * dim)
        latents = S.pop("latents")
        _tree(self, S)
        self.latents = nn.Parameter(torch.randn(latents) / math.sqrt(dim), requires_grad=False)
        self._packed = None

    @property
    def dtype(self):
        return self.latents.dtype

    @property
    def device(self):
        return self.latents.device

    def _apply(self, fn, *a, **k):
        self._packed = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._packed = None
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _pack(self):
        if self._packed is not None:
            return self._packed
        dev = self.device
        W: Dict[str, torch.Tensor] = {}
        for k, v in self.state_dict().items():
            v = v.detach().to(device=dev, dtype=BF16)                                  # model-dtype rounding
            W[k] = v.float().contiguous() if (v.dim() == 1 or k == "pos_emb.weight") else v.contiguous()
        for i in range(self.cfg["depth"]):
            f = f"layers.{i}.1"
            w1 = W[f + ".1.weight"]
            # GELU(h @ w1.T) through the GEGLU epilogue: value half = 0 * h + 1, gate half = w1
            wv = torch.cat([torch.zeros_like(w1), w1], 0)
            bv = torch.cat([torch.ones(w1.shape[0], device=dev), torch.zeros(w1.shape[0], device=dev)])
            W[f + ".gelu_w"], W[f + ".gelu_b"], _ = ops.pack_geglu(wv, bv)
        self._packed = W
        return W

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x (L, n <= max_seq_len, embedding_dim) -> (L, num_queries, output_dim) bf16 (reference :128-150)."""
        from .. import _ffi
        _ffi.require_sm90()
        c = self.cfg
        W = self._pack()
        dev = self.device
        L, n, E = x.shape
        D, nq, heads, inner = c["dim"], c["num_queries"], c["heads"], c["dim_head"] * c["heads"]
        xb = (x.to(device=dev, dtype=BF16) + W["pos_emb.weight"][:n].to(BF16)).reshape(L * n, E).contiguous()
        lat = W["latents"].reshape(nq, D).repeat(L, 1).contiguous()                   # (L*nq, D) bf16
        xf = ops.gemm(xb, W["proj_in.weight"], W["proj_in.bias"])
        for i in range(c["depth"]):
            a, f = f"layers.{i}.0", f"layers.{i}.1"
            xn = ops.layernorm(xf, W[a + ".norm1.weight"], W[a + ".norm1.bias"])
            ln = ops.layernorm(lat, W[a + ".norm2.weight"], W[a + ".norm2.bias"])
            q = ops.gemm(ln, W[a + ".to_q.weight"])
            kv_in = torch.cat([xn.view(L, n, D), ln.view(L, nq, D)], 1).reshape(L * (n + nq), D).contiguous()
            kv = ops.gemm(kv_in, W[a + ".to_kv.weight"])
            o = ops.flash_attention(q, kv[:, :inner], kv[:, inner:], heads, nq, n + nq)
            lat = ops.gemm(o, W[a + ".to_out.weight"], residual=lat)
            h = ops.layernorm(lat, W[f + ".0.weight"], W[f + ".0.bias"])
            g = ops.gemm(h, W[f + ".gelu_w"], W[f + ".gelu_b"], geglu=True)
            lat = ops.gemm(g, W[f + ".3.weight"], residual=lat)
        out = ops.gemm(lat, W["proj_out.weight"], W["proj_out.bias"])
        out = ops.layernorm(out, W["norm_out.weight"], W["norm_out.bias"])
        return out.view(L, nq, c["output_dim"])
