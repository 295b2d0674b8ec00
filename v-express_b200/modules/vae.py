"""H100-native VAE decoder: drop-in for the ``AutoencoderKL.decode`` the reference pipeline calls
(pipelines/v_express_pipeline.py:152-166; diffusers 0.29.2 AutoencoderKL with the sd-vae-ft-mse config,
SURVEY.md Appendix B.6).  Same ``state_dict`` keys as diffusers for ``post_quant_conv.*`` and ``decoder.*``
(encoder keys are accepted and ignored: VAE *encode* is outside the hot path, SURVEY.md 8f-f4).

All frames are decoded in ONE batch on the channels-last bf16 layout (the reference decodes frame by frame with
a device->host copy per frame): two-source-free GroupNorm+SiLU kernels, wgmma implicit-GEMM 3x3 convs with the
residual add in the epilogue, nearest-2x upsample, and the single-head hd=512 mid-block attention as
GEMM(QK^T, fp32 scores) -> row softmax -> GEMM(PV).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
from torch import nn

from .. import ops
from .unet_3d import _Config, _Node, _Norm

BF16 = torch.bfloat16


class DecoderOutput:
    def __init__(self, sample):
        self.sample = sample


class EncoderOutput:
    def __init__(self, latent_dist):
        self.latent_dist = latent_dist


class _MeanOnlyDistribution:
    """The part of diffusers' DiagonalGaussianDistribution the reference touches: ``.mean`` (and ``.mode()``)."""

    def __init__(self, mean):
        self.mean = mean

    def mode(self):
        return self.mean

    def sample(self, generator=None):
        raise NotImplementedError("only the posterior mean is computed (the reference uses latent_dist.mean)")


def _vae_keys(boc, layers, latent, out_ch) -> Dict[str, Tuple[int, ...]]:
    S: Dict[str, Tuple[int, ...]] = {}

    def wb(p, *shape):
        S[p + ".weight"] = tuple(shape)
        S[p + ".bias"] = (shape[0],)

    def res(p, ci, co):
        wb(p + ".norm1", ci)
        wb(p + ".conv1", co, ci, 3, 3)
        wb(p + ".norm2", co)
        wb(p + ".conv2", co, co, 3, 3)
        if ci != co:
            wb(p + ".conv_shortcut", co, ci, 1, 1)

    wb("post_quant_conv", latent, latent, 1, 1)
    d = "decoder"
    top = boc[-1]
    wb(d + ".conv_in", top, latent, 3, 3)
    res(d + ".mid_block.resnets.0", top, top)
    a = d + ".mid_block.attentions.0"
    wb(a + ".group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        wb(f"{a}.{n}", top, top)
    res(d + ".mid_block.resnets.1", top, top)
    rev = list(reversed(boc))
    co = rev[0]
    for i in range(len(boc)):
        ci, co = co, rev[i]
        for j in range(layers + 1):
            res(f"{d}.up_blocks.{i}.resnets.{j}", ci if j == 0 else co, co)
        if i < len(boc) - 1:
            wb(f"{d}.up_blocks.{i}.upsamplers.0.conv", co, co, 3, 3)
    wb(d + ".conv_norm_out", boc[0])
    wb(d + ".conv_out", out_ch, boc[0], 3, 3)
    return S


def _vae_encoder_keys(boc, layers, latent, in_ch) -> Dict[str, Tuple[int, ...]]:
    """``encoder.*`` + ``quant_conv.*`` of diffusers' AutoencoderKL (Encoder / DownEncoderBlock2D / UNetMidBlock2D)."""
    S: Dict[str, Tuple[int, ...]] = {}

    def wb(p, *shape):
        S[p + ".weight"] = tuple(shape)
        S[p + ".bias"] = (shape[0],)

    def res(p, ci, co):
        wb(p + ".norm1", ci)
        wb(p + ".conv1", co, ci, 3, 3)
        wb(p + ".norm2", co)
        wb(p + ".conv2", co, co, 3, 3)
        if ci != co:
            wb(p + ".conv_shortcut", co, ci, 1, 1)

    e = "encoder"
    wb(e + ".conv_in", boc[0], in_ch, 3, 3)
    co = boc[0]
    for i, ch in enumerate(boc):
        ci, co = co, ch
        for j in range(layers):
            res(f"{e}.down_blocks.{i}.resnets.{j}", ci if j == 0 else co, co)
        if i < len(boc) - 1:
            wb(f"{e}.down_blocks.{i}.downsamplers.0.conv", co, co, 3, 3)
    top = boc[-1]
    res(e + ".mid_block.resnets.0", top, top)
    a = e + ".mid_block.attentions.0"
    wb(a + ".group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        wb(f"{a}.{n}", top, top)
    res(e + ".mid_block.resnets.1", top, top)
    wb(e + ".conv_norm_out", top)
    wb(e + ".conv_out", 2 * latent, top, 3, 3)
    wb("quant_conv", 2 * latent, 2 * latent, 1, 1)
    return S


class AutoencoderKL(nn.Module):
    """Decoder half of diffusers' AutoencoderKL (parameters only; arithmetic on sm_90a kernels)."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, norm_num_groups=32, act_fn="silu", scaling_factor=0.18215, with_encoder=True,
                 **_ignored):
        super().__init__()
        if norm_num_groups != 32 or act_fn != "silu" or any(c % 64 for c in block_out_channels):
            raise ValueError("vexpress_b200.AutoencoderKL: unsupported configuration")
        self.config = _Config(in_channels=in_channels, out_channels=out_channels,
                              block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                              latent_channels=latent_channels, norm_num_groups=norm_num_groups,
                              scaling_factor=scaling_factor)
        keys = _vae_keys(tuple(block_out_channels), layers_per_block, latent_channels, out_channels)
        self.has_encoder = bool(with_encoder)
        if with_encoder:
            keys.update(_vae_encoder_keys(tuple(block_out_channels), layers_per_block, latent_channels, in_channels))
        for key, shape in keys.items():
            parts = key.split(".")
            node = self
            for depth, name in enumerate(parts[:-1]):
                child = node._modules.get(name)
                if child is None:
                    child = _Norm() if "norm" in name else _Node()
                    node.add_module(name, child)
                node = child
            node.register_parameter(parts[-1], nn.Parameter(torch.empty(shape), requires_grad=False))
        self._engine: Optional[VaeDecoderEngine] = None
        self._enc_engine: Optional["VaeEncoderEngine"] = None
        self._encoder_loaded = False

    @property
    def dtype(self):
        return self.post_quant_conv.weight.dtype

    @property
    def device(self):
        return self.post_quant_conv.weight.device

    def _apply(self, fn, *a, **k):
        self._engine = None
        self._enc_engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._engine = None
        self._enc_engine = None
        sd = {}
        # checkpoints saved before diffusers 0.18 (stabilityai/sd-vae-ft-mse among them) name the mid-block attention
        # projections query / key / value / proj_attn; diffusers renames them at load time
        # (AutoencoderKL._convert_deprecated_attention_blocks) -- same here
        old = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}
        has_enc = any(k.startswith("encoder.") for k in state_dict)
        for k, v in state_dict.items():
            if (k.startswith("encoder.") or k.startswith("quant_conv.")) and not self.has_encoder:
                continue
            if ".attentions." in k:
                for a, b in old.items():
                    if a in k:
                        k = k.replace(a, b)
                        if v.dim() == 4:
                            v = v.reshape(v.shape[0], v.shape[1])
            sd[k] = v
        if self.has_encoder and not has_enc:
            # decoder-only checkpoint (the hot path needs nothing else): the encoder parameters stay uninitialised and
            # ``encode`` refuses to run
            own = super().state_dict()
            sd.update({k: own[k] for k in own if k.startswith("encoder.") or k.startswith("quant_conv.")})
        else:
            self._encoder_loaded = self.has_encoder
        return super().load_state_dict(sd, strict=strict, **kw)

    def state_dict(self, *a, **k):
        sd = super().state_dict(*a, **k)
        if self.has_encoder and not self._encoder_loaded:
            for key in [key for key in sd if key.startswith("encoder.") or key.startswith("quant_conv.")]:
                del sd[key]
        return sd

    def engine(self) -> "VaeDecoderEngine":
        if self._engine is None:
            self._engine = VaeDecoderEngine(self)
        return self._engine

    @torch.no_grad()
    def encode(self, x, return_dict: bool = True):
        """x (n,3,H,W) in [-1,1] -> ``.latent_dist`` with ``.mean`` / ``.mode()`` (n,4,H/8,W/8) in the model dtype: what
        the reference's ``prepare_reference_latent`` reads (pipelines/v_express_pipeline.py:343-348).  Only the mean of
        the posterior is computed (``sample()`` is not offered: the reference never samples the reference latent)."""
        if not (self.has_encoder and self._encoder_loaded):
            raise RuntimeError("vexpress_b200.AutoencoderKL.encode: no encoder weights were loaded (decoder-only checkpoint)")
        if self._enc_engine is None:
            self._enc_engine = VaeEncoderEngine(self)
        mean = self._enc_engine.encode_mean(x.to(BF16)).to(x.dtype)
        dist = _MeanOnlyDistribution(mean)
        return EncoderOutput(dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z, return_dict: bool = True):
        """z (n,4,h,w), already divided by the scaling factor by the caller -> sample (n,3,8h,8w), model dtype."""
        out = self.engine().decode(z.to(BF16), pre_scale=1.0, post=False, out_dtype=BF16).to(z.dtype)
        return DecoderOutput(out) if return_dict else (out,)

    @torch.no_grad()
    def decode_latents(self, latents, out=None):
        """Fused form of the reference's ``decode_latents`` (pipelines/v_express_pipeline.py:152-166):
        latents (n,4,h,w) UNSCALED -> fp32 frames (n,3,8h,8w) in [0,1] on the device.  ``out``: optional fp32 view of
        that shape whose (h, w) planes are contiguous (frame / channel strides are free)."""
        return self.engine().decode(latents.to(BF16), pre_scale=1.0 / self.config["scaling_factor"], post=True,
                                    out_dtype=torch.float32, out=out)


class VaeDecoderEngine:
    def __init__(self, model: AutoencoderKL):
        from .. import _ffi
        _ffi.require_sm90()
        if model.device.type != "cuda":
            raise RuntimeError("vexpress_b200: the VAE must live on a CUDA (sm_90a) device; there is no CPU path")
        _ffi.note_compute_dtype(model.dtype, "AutoencoderKL")
        self.model = model
        self.dev = model.device
        self.boc = tuple(model.config["block_out_channels"])
        self.layers = model.config["layers_per_block"]
        self.W: Dict[str, torch.Tensor] = {}
        self._pack({k: v for k, v in nn.Module.state_dict(model).items()
                    if not (k.startswith("encoder.") or k.startswith("quant_conv."))})

    def _pack(self, msd):
        """The decoder parameters of ``msd`` (``post_quant_conv.*``, ``decoder.*``) in the kernels' layouts, into ``self.W``
        on ``self.dev``.  Host-side tensor operations only (no kernel is launched), so it also packs on the CPU or the meta
        device."""
        dev = self.dev
        self.W.update(ops.f32_arena({k: v for k, v in msd.items() if k.endswith(".bias") or v.dim() == 1}, dev))
        for k, v in msd.items():
            v = v.detach()
            p = k.rsplit(".", 1)[0]
            if k.endswith(".bias") or v.dim() == 1:
                continue
            elif p == "decoder.conv_in":
                self.W[k] = v.to(device=dev, dtype=BF16).float().reshape(v.shape[0], -1).t().contiguous()
            elif p == "decoder.conv_out":
                self.W["conv_out.packed_w"], self.W["conv_out.packed_b"] = ops.pack_conv_out(
                    v.to(device=dev, dtype=BF16), self.W[p + ".bias"])
            elif p == "post_quant_conv":
                self.W[k] = v.to(device=dev, dtype=BF16).float().reshape(v.shape[0], v.shape[1]).contiguous()
            elif v.dim() == 4 and v.shape[-1] == 3 and ".upsamplers." in k:
                self.W[k] = ops.pack_upconv_weight(v.to(device=dev, dtype=BF16))    # upsample folded into the conv
            elif v.dim() == 4 and v.shape[-1] == 3:
                self.W[k] = ops.pack_conv3x3_weight(v.to(device=dev, dtype=BF16))
            elif v.dim() == 4:
                self.W[k] = v.to(device=dev, dtype=BF16).reshape(v.shape[0], v.shape[1]).contiguous()
            else:
                self.W[k] = v.to(device=dev, dtype=BF16).contiguous()

    def _res(self, p, x, NB, H, Wd):
        W = self.W
        h = ops.groupnorm(x, NB, H * Wd, W[p + ".norm1.weight"], W[p + ".norm1.bias"], 1e-6, True)
        h = ops.conv3x3(h.view(NB, H, Wd, -1), W[p + ".conv1.weight"], W[p + ".conv1.bias"])
        h = ops.groupnorm(h, NB, H * Wd, W[p + ".norm2.weight"], W[p + ".norm2.bias"], 1e-6, True)
        sc = x
        if (p + ".conv_shortcut.weight") in W:
            sc = ops.gemm(x, W[p + ".conv_shortcut.weight"], W[p + ".conv_shortcut.bias"])
        return ops.conv3x3(h.view(NB, H, Wd, -1), W[p + ".conv2.weight"], W[p + ".conv2.bias"], residual=sc)

    def _attn(self, p, x, NB, HW):
        """Single-head attention over the HW tokens of each frame (diffusers Attention with group_norm,
        biased projections, residual connection)."""
        W = self.W
        C = x.shape[1]
        xn = ops.groupnorm(x, NB, HW, W[p + ".group_norm.weight"], W[p + ".group_norm.bias"], 1e-6, False)
        q = ops.gemm(xn, W[p + ".to_q.weight"], W[p + ".to_q.bias"])
        k = ops.gemm(xn, W[p + ".to_k.weight"], W[p + ".to_k.bias"])
        o = torch.empty_like(q)
        scores = torch.empty((HW, HW), device=self.dev, dtype=torch.float32)
        probs = torch.empty((HW, HW), device=self.dev, dtype=BF16)
        vt = torch.empty((C, HW), device=self.dev, dtype=BF16)
        for n in range(NB):
            sl = slice(n * HW, (n + 1) * HW)
            ops.gemm(q[sl], k[sl], scale=C ** -0.5, out=scores, out_f32=True)
            ops.softmax_rows(scores, out=probs)
            # V^T = Wv @ xn^T (bias added after P@V: softmax rows sum to 1, so P (V + 1 b^T) = P V + b^T)
            ops.gemm(W[p + ".to_v.weight"], xn[sl], out=vt)
            ops.gemm(probs, vt, W[p + ".to_v.bias"], out=o[sl])
        return ops.gemm(o, W[p + ".to_out.0.weight"], W[p + ".to_out.0.bias"], residual=x)

    def decode(self, z, pre_scale: float, post: bool, out_dtype, out=None):
        W = self.W
        assert z.dim() == 4
        z = z.contiguous()
        NB, _, H, Wd = z.shape
        d = "decoder"
        x = ops.conv_in(z, W[d + ".conv_in.weight"], W[d + ".conv_in.bias"], self.boc[-1], pre_scale=pre_scale,
                        pre_w=W["post_quant_conv.weight"], pre_b=W["post_quant_conv.bias"])
        x = self._res(d + ".mid_block.resnets.0", x, NB, H, Wd)
        x = self._attn(d + ".mid_block.attentions.0", x, NB, H * Wd)
        x = self._res(d + ".mid_block.resnets.1", x, NB, H, Wd)
        nb = len(self.boc)
        for i in range(nb):
            for j in range(self.layers + 1):
                x = self._res(f"{d}.up_blocks.{i}.resnets.{j}", x, NB, H, Wd)
            if i < nb - 1:
                x = ops.upconv3x3(x.view(NB, H, Wd, -1), W[f"{d}.up_blocks.{i}.upsamplers.0.conv.weight"],
                                  W[f"{d}.up_blocks.{i}.upsamplers.0.conv.bias"])
                H, Wd = 2 * H, 2 * Wd
        x = ops.groupnorm(x, NB, H * Wd, W[d + ".conv_norm_out.weight"], W[d + ".conv_norm_out.bias"], 1e-6, True)
        if out is None:
            out = torch.empty((NB, self.model.config["out_channels"], H, Wd), device=self.dev, dtype=out_dtype)
        assert out.shape == (NB, self.model.config["out_channels"], H, Wd) and out.dtype == out_dtype
        ops.conv_out_tc(x, NB, H, Wd, W["conv_out.packed_w"], W["conv_out.packed_b"], out, post=post)
        return out


class VaeEncoderEngine:
    """``AutoencoderKL.encode(x).latent_dist.mean`` (diffusers Encoder: conv_in 3->128, DownEncoderBlock2D x4 with the
    pad-(0,1,0,1) stride-2 downsamplers, UNetMidBlock2D with the single-head attention, GroupNorm -> SiLU -> conv_out,
    quant_conv) on the decoder's kernels -- SURVEY.md 8(f) row f4.  Runs once per video on one 512x512 image.
    ``quant_conv`` (1x1, linear) is folded into ``conv_out`` on the host and only the 4 mean channels are produced."""

    def __init__(self, model: AutoencoderKL):
        from .. import _ffi
        _ffi.require_sm90()
        if model.device.type != "cuda":
            raise RuntimeError("vexpress_b200: the VAE must live on a CUDA (sm_90a) device; there is no CPU path")
        _ffi.note_compute_dtype(model.dtype, "AutoencoderKL")
        self.model = model
        self.dev = dev = model.device
        self.boc = tuple(model.config["block_out_channels"])
        self.layers = model.config["layers_per_block"]
        lc = model.config["latent_channels"]
        sd = {k: v.detach() for k, v in nn.Module.state_dict(model).items() if k.startswith("encoder.") or k.startswith("quant_conv.")}
        self.W: Dict[str, torch.Tensor] = {}
        self.W.update(ops.f32_arena({k: v for k, v in sd.items() if k.endswith(".bias") or v.dim() == 1}, dev))
        bf = lambda t: t.to(device=dev, dtype=BF16)
        for k, v in sd.items():
            p = k.rsplit(".", 1)[0]
            if k.endswith(".bias") or v.dim() == 1 or p in ("quant_conv", "encoder.conv_out"):
                continue
            if p == "encoder.conv_in":
                w4 = torch.zeros((v.shape[0], 4, 3, 3), device=dev, dtype=torch.float32)      # RGB + one zero channel
                w4[:, :v.shape[1]] = bf(v).float()
                self.W[k] = w4.reshape(v.shape[0], -1).t().contiguous()                     # fp32 [4*9, Cout]
            elif v.dim() == 4 and v.shape[-1] == 3:
                self.W[k] = ops.pack_conv3x3_weight(bf(v))
            elif v.dim() == 4:
                self.W[k] = bf(v).reshape(v.shape[0], v.shape[1]).contiguous()
            else:
                self.W[k] = bf(v).contiguous()
        # mean = quant_conv(conv_out(h))[:, :lc]: fold the 1x1 into the 3x3 (both linear), keep the mean rows only
        q = bf(sd["quant_conv.weight"]).float().reshape(2 * lc, 2 * lc)[:lc]                  # (lc, 2lc)
        wo = bf(sd["encoder.conv_out.weight"]).float()                                       # (2lc, C, 3, 3)
        w_fold = torch.einsum("om,mckl->ockl", q, wo)
        b_fold = q @ bf(sd["encoder.conv_out.bias"]).float() + bf(sd["quant_conv.bias"]).float()[:lc]
        self.W["mean.packed_w"], self.W["mean.packed_b"] = ops.pack_conv_out(w_fold.to(BF16), b_fold)
        self.lc = lc

    _res = VaeDecoderEngine._res
    _attn = VaeDecoderEngine._attn

    def encode_mean(self, x):
        W = self.W
        assert x.dim() == 4 and x.shape[1] == 3
        NB, _, H, Wd = x.shape
        if H % 8 or Wd % 8:
            raise ValueError(f"image size {H}x{Wd} must be a multiple of 8")
        x4 = torch.zeros((NB, 4, H, Wd), device=self.dev, dtype=BF16)
        x4[:, :3] = x.to(device=self.dev, dtype=BF16)
        e = "encoder"
        h = ops.conv_in(x4, W[e + ".conv_in.weight"], W[e + ".conv_in.bias"], self.boc[0])
        for i in range(len(self.boc)):
            for j in range(self.layers):
                h = self._res(f"{e}.down_blocks.{i}.resnets.{j}", h, NB, H, Wd)
            if i < len(self.boc) - 1:
                # Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) then conv3x3 stride 2
                h = ops.downsample_conv(h, NB, H, Wd, W[f"{e}.down_blocks.{i}.downsamplers.0.conv.weight"],
                                        W[f"{e}.down_blocks.{i}.downsamplers.0.conv.bias"], pad_lo=0)
                H, Wd = H // 2, Wd // 2
        h = self._res(e + ".mid_block.resnets.0", h, NB, H, Wd)
        h = self._attn(e + ".mid_block.attentions.0", h, NB, H * Wd)
        h = self._res(e + ".mid_block.resnets.1", h, NB, H, Wd)
        h = ops.groupnorm(h, NB, H * Wd, W[e + ".conv_norm_out.weight"], W[e + ".conv_norm_out.bias"], 1e-6, True)
        out = torch.empty((NB, self.lc, H, Wd), device=self.dev, dtype=BF16)
        ops.conv_out_tc(h, NB, H, Wd, W["mean.packed_w"], W["mean.packed_b"], out)
        return out
