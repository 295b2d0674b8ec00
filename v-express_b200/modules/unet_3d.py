"""H100-native denoising UNet: drop-in for the reference's ``modules/unet_3d.py``.

Same constructor configuration, ``state_dict`` key/shape layout (SURVEY.md Appendix C; 1386 tensors at full
width) and ``forward`` signature as the reference ``UNet3DConditionModel`` (modules/unet_3d.py:30-250, 400-578),
but the module tree holds parameters only: the arithmetic is executed by hand-written sm_90a kernels through
the C ABI (``vexpress_b200.ops``) on a channels-last bf16 token layout ``[(b f)(h w), C]``:

* ResnetBlock3D (modules/resnet.py:217-251): two-source GroupNorm+SiLU -> wgmma implicit-GEMM 3x3 conv with
  bias + time-embedding + residual epilogues; the skip ``torch.cat`` (unet_3d_blocks.py:694,831) is folded
  into the GroupNorm read and the split-K of the 1x1 shortcut GEMM;
* Transformer3DModel + read-mode TemporalBasicTransformerBlock (modules/transformer_3d.py:103-169,
  modules/mutual_self_attention.py:176-267): GEMMs with fused bias/scale/residual epilogues, wgmma flash
  attention for attn1 and attn1_5 (bank K/V projected ONCE per bank instead of per frame per step), 5-token
  audio attention kernel, GEGLU;
* VanillaTemporalModule (modules/motion_module.py:44-388): temporal attention reads the (b f)(h w) layout with a
  frame stride, positional encoding fused into the LayerNorm.

There is no PyTorch/CPU fallback: ``forward`` raises if the CUDA library is missing.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from .. import ops

BF16 = torch.bfloat16


# ----------------------------------------------------------------------------------------------
# configuration + parameter layout
# ----------------------------------------------------------------------------------------------
@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class _Config(dict):
    __getattr__ = dict.__getitem__


_DOWN = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D")
_UP = ("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D")


def _unet_keys(boc, cross, layers, in_ch, out_ch, pe_len) -> Dict[str, Tuple[int, ...]]:
    """state_dict key -> shape (the weight contract, SURVEY.md Appendix C)."""
    S: Dict[str, Tuple[int, ...]] = {}
    ted = boc[0] * 4

    def wb(p, *shape):
        S[p + ".weight"] = tuple(shape)
        S[p + ".bias"] = (shape[0],)

    def attn(p, c, kv):
        S[p + ".to_q.weight"] = (c, c)
        S[p + ".to_k.weight"] = (c, kv)
        S[p + ".to_v.weight"] = (c, kv)
        wb(p + ".to_out.0", c, c)

    def ff(p, c):
        wb(p + ".net.0.proj", 8 * c, c)
        wb(p + ".net.2", c, 4 * c)

    def resnet(p, ci, co):
        wb(p + ".norm1", ci)
        wb(p + ".conv1", co, ci, 3, 3)
        wb(p + ".time_emb_proj", co, ted)
        wb(p + ".norm2", co)
        wb(p + ".conv2", co, co, 3, 3)
        if ci != co:
            wb(p + ".conv_shortcut", co, ci, 1, 1)

    def spatial(p, c):
        wb(p + ".norm", c)
        wb(p + ".proj_in", c, c, 1, 1)
        t = p + ".transformer_blocks.0"
        for name, kv in (("attn1", c), ("attn1_5", c), ("attn2", cross)):
            attn(f"{t}.{name}", c, kv)
        for name in ("norm1", "norm1_5", "norm2", "norm3"):
            wb(f"{t}.{name}", c)
        ff(t + ".ff", c)
        wb(p + ".proj_out", c, c, 1, 1)

    def motion(p, c):
        p += ".temporal_transformer"
        wb(p + ".norm", c)
        wb(p + ".proj_in", c, c)
        t = p + ".transformer_blocks.0"
        for i in (0, 1):
            attn(f"{t}.attention_blocks.{i}", c, c)
            S[f"{t}.attention_blocks.{i}.pos_encoder.pe"] = (1, pe_len, c)
            wb(f"{t}.norms.{i}", c)
        ff(t + ".ff", c)
        wb(t + ".ff_norm", c)
        wb(p + ".proj_out", c, c)

    wb("conv_in", boc[0], in_ch, 3, 3)
    wb("time_embedding.linear_1", ted, boc[0])
    wb("time_embedding.linear_2", ted, ted)
    co = boc[0]
    for i in range(4):
        ci, co = co, boc[i]
        for j in range(layers):
            resnet(f"down_blocks.{i}.resnets.{j}", ci if j == 0 else co, co)
            if i < 3:
                spatial(f"down_blocks.{i}.attentions.{j}", co)
            motion(f"down_blocks.{i}.motion_modules.{j}", co)
        if i < 3:
            wb(f"down_blocks.{i}.downsamplers.0.conv", co, co, 3, 3)
    c = boc[-1]
    resnet("mid_block.resnets.0", c, c)
    spatial("mid_block.attentions.0", c)
    motion("mid_block.motion_modules.0", c)
    resnet("mid_block.resnets.1", c, c)
    rev = list(reversed(boc))
    co = rev[0]
    for i in range(4):
        prev, co = co, rev[i]
        ci = rev[min(i + 1, 3)]
        for j in range(layers + 1):
            skip = ci if j == layers else co
            resnet(f"up_blocks.{i}.resnets.{j}", (prev if j == 0 else co) + skip, co)
            if i > 0:
                spatial(f"up_blocks.{i}.attentions.{j}", co)
            motion(f"up_blocks.{i}.motion_modules.{j}", co)
        if i < 3:
            wb(f"up_blocks.{i}.upsamplers.0.conv", co, co, 3, 3)
    wb("conv_norm_out", boc[0])
    wb("conv_out", out_ch, boc[0], 3, 3)
    return S


class _Node(nn.Module):
    """Parameter container; children are attached under the reference's attribute names."""


class _Norm(_Node):
    @property
    def normalized_shape(self):
        return (self.weight.shape[0],)


class TemporalBasicTransformerBlock(_Node):
    """Parameter holder of one spatial transformer block + the per-block reference ``bank``
    (reference modules/attention.py:298-395; hooks modules/mutual_self_attention.py:286-319)."""

    def __init__(self):
        super().__init__()
        self.bank: List[torch.Tensor] = []


def _positional_encoding(d_model: int, max_len: int) -> torch.Tensor:
    """Sinusoidal table of the temporal attention (reference modules/motion_module.py:262-273)."""
    pos = torch.arange(max_len, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(1, max_len, d_model)
    pe[0, :, 0::2] = torch.sin(pos * div)
    pe[0, :, 1::2] = torch.cos(pos * div)
    return pe


def _build_tree(root: nn.Module, shapes: Dict[str, Tuple[int, ...]]):
    for key, shape in shapes.items():
        parts = key.split(".")
        node = root
        for depth, name in enumerate(parts[:-1]):
            child = node._modules.get(name)
            if child is None:
                path = parts[:depth + 1]
                if name == "0" and len(path) >= 2 and path[-2] == "transformer_blocks" and "attentions" in path:
                    child = TemporalBasicTransformerBlock()
                elif "norm" in name or (len(path) >= 2 and path[-2] == "norms"):
                    child = _Norm()
                else:
                    child = _Node()
                node.add_module(name, child)
            node = child
        leaf = parts[-1]
        if leaf == "pe":
            node.register_buffer("pe", _positional_encoding(shape[2], shape[1]))
        else:
            node.register_parameter(leaf, nn.Parameter(torch.empty(shape), requires_grad=False))


def attention_block_order(model: "UNet3DConditionModel") -> List[str]:
    """Reader-block pairing order of ``ReferenceAttentionControl.update``: depth-first module order
    (down_blocks, up_blocks, mid_block -- registration order of the reference, see unet_3d.py:108-160),
    stable-sorted by descending width (modules/mutual_self_attention.py:346-351)."""
    mods = dict(model.named_modules())
    dfs = [f"down_blocks.{i}.attentions.{j}" for i in range(3) for j in range(2)]
    dfs += [f"up_blocks.{i}.attentions.{j}" for i in (1, 2, 3) for j in range(3)]
    dfs += ["mid_block.attentions.0"]
    names = [n + ".transformer_blocks.0" for n in dfs]
    assert all(isinstance(mods[n], TemporalBasicTransformerBlock) for n in names)
    return sorted(names, key=lambda n: -mods[n].norm1.normalized_shape[0])


# ----------------------------------------------------------------------------------------------
# the model (parameters + public API)
# ----------------------------------------------------------------------------------------------
class UNet3DConditionModel(nn.Module):
    def __init__(self, sample_size=None, in_channels=4, out_channels=4, center_input_sample=False,
                 flip_sin_to_cos=True, freq_shift=0, down_block_types=_DOWN, mid_block_type="UNetMidBlock3DCrossAttn",
                 up_block_types=_UP, only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280),
                 layers_per_block=2, downsample_padding=1, mid_block_scale_factor=1, act_fn="silu",
                 norm_num_groups=32, norm_eps=1e-5, cross_attention_dim=1280, attention_head_dim=8,
                 dual_cross_attention=False, use_linear_projection=False, class_embed_type=None,
                 num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift="default",
                 use_inflated_groupnorm=False, use_motion_module=False, motion_module_resolutions=(1, 2, 4, 8),
                 motion_module_mid_block=False, motion_module_decoder_only=False, motion_module_type=None,
                 motion_module_kwargs=None, unet_use_cross_frame_attention=None, unet_use_temporal_attention=None):
        super().__init__()
        mmk = dict(motion_module_kwargs or {})
        cfg = dict(locals())
        for k in ("self", "__class__", "mmk", "cfg"):
            cfg.pop(k, None)
        cfg["motion_module_kwargs"] = mmk
        self.config = _Config(cfg)
        self.sample_size = sample_size

        # this build implements exactly the inference configuration of inference_v2.yaml:1-21 on the SD-1.5
        # topology; anything else is rejected loudly rather than silently approximated
        def need(cond, what):
            if not cond:
                raise ValueError(f"vexpress_b200.UNet3DConditionModel: unsupported configuration: {what}")
        if mid_block_type != "UNetMidBlock3DCrossAttn":
            raise ValueError(f"unknown mid_block_type : {mid_block_type}")
        need(tuple(down_block_types) == _DOWN and tuple(up_block_types) == _UP, "block types")
        need(len(block_out_channels) == 4 and layers_per_block == 2, "4 levels x 2 layers")
        need(act_fn in ("silu", "swish") and norm_num_groups == 32 and resnet_time_scale_shift == "default", "act/norm")
        need(not center_input_sample and flip_sin_to_cos and freq_shift == 0, "time projection")
        need(not dual_cross_attention and not use_linear_projection and class_embed_type is None
             and num_class_embeds is None and not only_cross_attention and not upcast_attention, "attention flags")
        need(use_inflated_groupnorm and use_motion_module and motion_module_mid_block
             and not motion_module_decoder_only and motion_module_type == "Vanilla"
             and tuple(motion_module_resolutions) == (1, 2, 4, 8), "motion-module placement")
        need(not unet_use_temporal_attention and not unet_use_cross_frame_attention, "unet temporal/cross-frame attn")
        need(mmk.get("num_attention_heads", 8) == 8 and mmk.get("num_transformer_block", 2) == 1
             and tuple(mmk.get("attention_block_types", ())) == ("Temporal_Self", "Temporal_Self")
             and mmk.get("temporal_position_encoding", False) and mmk.get("temporal_attention_dim_div", 1) == 1,
             "motion_module_kwargs")
        need(attention_head_dim == 8 or tuple(attention_head_dim) == (8, 8, 8, 8), "attention_head_dim (= #heads) 8")
        need(all(c % 64 == 0 for c in block_out_channels), "channel widths must be multiples of 64")
        self.heads = 8
        self.pe_len = int(mmk.get("temporal_position_encoding_max_len", 24))
        _build_tree(self, _unet_keys(tuple(block_out_channels), cross_attention_dim, layers_per_block, in_channels,
                                     out_channels, self.pe_len))
        self._engine: Optional[UNetEngine] = None
        self._fp8_linear = False
        self.reference_attention_weight = 1.0
        self.audio_attention_weight = 1.0

    # ---- diffusers-style conveniences the reference callers use (inference.py:197-198, pipeline :468)
    @property
    def in_channels(self):
        return self.config["in_channels"]

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    @classmethod
    def load_config(cls, path):
        with open(path) as f:
            return json.load(f)

    @classmethod
    def from_config(cls, config, **kwargs):
        import inspect
        sig = inspect.signature(cls.__init__).parameters
        init = {k: v for k, v in dict(config).items() if k in sig}
        init.update({k: v for k, v in kwargs.items() if k in sig})
        return cls(**init)

    @classmethod
    def from_config_2d(cls, unet_config_path, unet_additional_kwargs=None):
        """Reference modules/unet_3d.py:673-698: SD-1.5 2-D config + forced 3-D block types."""
        cfg = cls.load_config(unet_config_path)
        cfg["_class_name"] = cls.__name__
        cfg["down_block_types"] = list(_DOWN)
        cfg["up_block_types"] = list(_UP)
        cfg["mid_block_type"] = "UNetMidBlock3DCrossAttn"
        return cls.from_config(cfg, **(unet_additional_kwargs or {}))

    def _apply(self, fn, *a, **k):
        self._engine = None  # parameters moved / cast: repack lazily
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._engine = None
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def engine(self) -> "UNetEngine":
        if self._engine is None:
            self._engine = UNetEngine(self)
        return self._engine

    # ---- opt-in FP8 (e4m3) for the Linears that read a LayerNorm output (DESIGN section 3, "FP8 mode")
    def enable_fp8_linear(self):
        """Run every Linear fed by a LayerNorm -- the fused q|k|v, attn1_5.to_q, attn2.to_q and the GEGLU projection of the
        spatial transformer blocks, the fused q|k|v and the GEGLU projection of the motion modules -- on e4m3 operands: the
        LayerNorm writes e4m3 codes with one scale per row, the weights are quantised per output channel.  Lossy (about 7.5 %
        relative L2 error of the noise prediction on the reduced-width test UNet, against 0.5 % for bf16): off by default.
        The e4m3 weights are packed next to the bf16 ones and rebuilt on every load_state_dict / .to."""
        _check_fp8_env()
        self._fp8_linear = True
        if self._engine is not None:
            self._engine.set_fp8(True)
        return self

    def disable_fp8_linear(self):
        """Back to the bf16 path (bit-identical to a model that never enabled FP8)."""
        self._fp8_linear = False
        if self._engine is not None:
            self._engine.set_fp8(False)
        return self

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, kps_features=None,
                attention_mask=None, down_block_additional_residuals=None, mid_block_additional_residual=None,
                return_dict: bool = True):
        """Reference signature (modules/unet_3d.py:400-411).  sample (b,4,f,h,w); encoder_hidden_states
        ((b f),5,768); kps_features (b,C0,f,h,w).  Returns sample (b,4,f,h,w) in the model dtype."""
        if class_labels is not None or attention_mask is not None or down_block_additional_residuals is not None \
                or mid_block_additional_residual is not None:
            raise ValueError("class_labels / attention_mask / additional residuals are not used on the V-Express "
                             "inference path and are not supported")
        assert sample.dim() == 5, f"Expected sample to have ndim=5, but got ndim={sample.dim()}."
        b, c, f, h, w = sample.shape
        eng = self.engine()
        frames = sample.to(BF16).permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w).contiguous()
        kps = None
        if kps_features is not None:
            kps = kps_features.to(BF16).permute(0, 2, 3, 4, 1).reshape(b * f * h * w, -1).contiguous()
        enc = encoder_hidden_states
        if enc.shape[0] != b * f:
            enc = enc.repeat_interleave(f, dim=0)
        out = eng.forward_frames(frames, timestep, enc, kps, None, b, f)            # ((b f), 4, h, w)
        out = out.view(b, f, -1, h, w).permute(0, 2, 1, 3, 4).to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)


def _check_fp8_env():
    for var in ("VX_LN_FOLD", "VX_LN_FUSE"):
        if os.environ.get(var, "0") not in ("", "0"):
            raise ValueError(f"enable_fp8_linear: {var} is set; that path normalises inside a bf16 GEMM, which has no "
                             f"e4m3 form -- unset it to use FP8")


# Linears that read a LayerNorm output (engine weight keys): the FP8 mode's coverage
_FP8_KEYS = (".qkv", ".attn1_5.to_q.weight", ".attn2.to_q.weight", ".ff.net.0.proj.geglu_w")


# ----------------------------------------------------------------------------------------------
# the engine: packed weights + kernel schedule
# ----------------------------------------------------------------------------------------------
class UNetEngine:
    """Owns the packed (kernel-layout) weights of one model instance and runs the forward schedule."""

    fp8 = False   # FP8 mode, off unless set_fp8(True) (the dry-run tests build engines without __init__)

    def __init__(self, model: UNet3DConditionModel):
        from .. import _ffi
        _ffi.require_sm90()
        dev = model.device
        if dev.type != "cuda":
            raise RuntimeError("vexpress_b200: the model must live on a CUDA (sm_90a) device; there is no CPU path")
        _ffi.note_compute_dtype(model.dtype, "UNet3DConditionModel")
        self.model = model
        self.dev = dev
        cfg = model.config
        self.boc = tuple(cfg["block_out_channels"])
        self.heads = model.heads
        self.groups = cfg["norm_num_groups"]
        self.eps = float(cfg["norm_eps"])
        self.cross = cfg["cross_attention_dim"]
        sd = {k: v.detach() for k, v in model.state_dict().items()}
        self.sd = sd
        self.W: Dict[str, torch.Tensor] = {}
        self._pack(sd)
        self._pack_ln_fold()
        self.W8: Dict[str, tuple] = {}            # the e4m3 weights, packed on first use of the FP8 mode
        self.set_fp8(model._fp8_linear)
        self._bank_cache: Dict[str, tuple] = {}
        self._bank_buf: Dict[str, torch.Tensor] = {}
        self._bank_flag: Dict[str, bool] = {}
        self.bank_epoch = 0
        self.order = attention_block_order(model)

    # ---------------------------------------------------------------- packing
    def _bf(self, t):
        return t.to(device=self.dev, dtype=BF16).contiguous()

    def _f32(self, t):
        # parameters are rounded to the model dtype first (what `.to(bf16)` does to the reference), then widened
        return t.to(device=self.dev, dtype=BF16).float().contiguous()

    def _pack(self, sd):
        W = self.W
        temb_w, temb_b, self.temb_off = [], [], {}
        off = 0
        W.update(ops.f32_arena({k: v for k, v in sd.items()
                                if k.endswith(".bias") or (k.endswith(".weight") and v.dim() == 1)}, self.dev))
        for k, v in sd.items():
            if not k.endswith(".weight") or v.dim() == 1:
                continue
            p = k[:-7]
            if p in ("conv_in",):
                W[k] = self._f32(v).reshape(v.shape[0], -1).t().contiguous()                 # fp32 [Cin*9, Cout]
            elif p == "conv_out":
                W["conv_out.packed_w"], W["conv_out.packed_b"] = ops.pack_conv_out(self._bf(v), W[p + ".bias"])
            elif p.endswith("time_emb_proj"):
                self.temb_off[p] = (off, v.shape[0])
                off += v.shape[0]
                temb_w.append(self._bf(v))
                temb_b.append(W[p + ".bias"])
            elif v.dim() == 4 and v.shape[-1] == 3 and ".upsamplers." in k:
                # nearest-2x upsample folded into the conv: four parity-class 2x2 kernels (ops.pack_upconv_weight)
                W[k] = ops.pack_upconv_weight(self._bf(v))
            elif v.dim() == 4 and v.shape[-1] == 3:
                W[k] = ops.pack_conv3x3_weight(self._bf(v))
            elif v.dim() == 4:
                W[k] = self._bf(v).reshape(v.shape[0], v.shape[1]).contiguous()              # 1x1 conv
            else:
                W[k] = self._bf(v)
        W["temb_cat.weight"] = torch.cat(temb_w, 0).contiguous()
        W["temb_cat.bias"] = torch.cat(temb_b, 0).contiguous()
        # fused projections
        for k in list(sd):
            if k.endswith("attn1.to_q.weight") or (k.endswith(".to_q.weight") and "attention_blocks" in k):
                p = k[:-len(".to_q.weight")]
                W[p + ".qkv"] = torch.cat([W[p + ".to_q.weight"], W[p + ".to_k.weight"], W[p + ".to_v.weight"]], 0).contiguous()
            elif k.endswith("attn1_5.to_q.weight") or k.endswith("attn2.to_q.weight"):
                p = k[:-len(".to_q.weight")]
                W[p + ".kv"] = torch.cat([W[p + ".to_k.weight"], W[p + ".to_v.weight"]], 0).contiguous()
            elif k.endswith("pos_encoder.pe"):
                W[k] = sd[k].to(device=self.dev, dtype=BF16).float()[0].contiguous()          # [max_len, C]
            elif k.endswith("ff.net.0.proj.weight"):
                p = k[:-len(".weight")]
                W[p + ".geglu_w"], W[p + ".geglu_b"], _ = ops.pack_geglu(W[k], W[p + ".bias"])

    # ---------------------------------------------------------------- LayerNorm folded into the consumer GEMM
    def _pack_ln_fold(self):
        """VX_LN_FOLD=1 (experiment, measured: parity green, no gain -- stays off): the LayerNorm -> Linear pairs of the
        transformer blocks as vx_row_stats + ops.gemm_lnfold (normalisation applied in the GEMM epilogue,
        ops.fold_layernorm), so LayerNorm(x) is never written to HBM.
        The one-kernel variant (ops.gemm_ln: row tile resident in shared memory, statistics computed in the kernel) passes
        its operator tests but is not wired into the engine (it was slower than LayerNorm kernel + GEMM at the 320-wide
        level when measured).
        Validated domain of both modes (tests/test_lnfold_bounds_gpu.py): LayerNorm input rows with |mean| / sigma <=
        R(K) = 0.8 * 2^12 / (K + 2) (10.2, 5.1, 2.6 at K = 320, 640, 1280) meet the default path's fp64 accuracy bound; the
        synthetic UNets stay below 0.6.  Beyond R the fold's uncentred accumulation and the hand-over's E[x^2] - mean^2
        variance (relative rstd error ~ 1.5 (nparts + 2) 2^-24 (mean / sigma)^2, unbounded on near-constant rows) void that
        guarantee; measured, both stayed at the default path's accuracy up to |mean| / sigma ~ 64."""
        self.ln_fold = os.environ.get("VX_LN_FOLD") == "1"
        # VX_LN_FUSE=1 (experiment, measured: parity green, SLOWER -- stays off): statistics hand-over.  Every LayerNorm
        # input is the output of a Linear (+ residual); that GEMM's epilogue emits per-row partial sums (ops.gemm_rowsums),
        # the consumer GEMM normalises in its epilogue (ops.gemm_lnparts): no LayerNorm kernel, no statistics kernel,
        # LayerNorm(x) never written.  The normalising epilogue costs more than the LayerNorm kernel it removes: the K = 320
        # / 640 GEMMs are bound by their epilogues' instruction issue.
        self.ln_fuse = os.environ.get("VX_LN_FUSE", "0") != "0" and not self.ln_fold
        self.F: Dict[str, tuple] = {}
        self._pe_proj: Dict[str, torch.Tensor] = {}
        self._pe_bias: Dict[tuple, torch.Tensor] = {}
        if not (self.ln_fold or self.ln_fuse):
            return
        W = self.W
        for k in list(W):
            if k.endswith(".norm1.weight") and ".attentions." in k:
                t = k[:-len(".norm1.weight")]
                for norm, lin in (("norm1", "attn1.qkv"), ("norm1_5", "attn1_5.to_q.weight"), ("norm2", "attn2.to_q.weight")):
                    if (t + "." + lin) in W:
                        self.F[f"{t}.{norm}"] = ops.fold_layernorm(W[f"{t}.{lin}"], None, W[f"{t}.{norm}.weight"],
                                                                   W[f"{t}.{norm}.bias"])
                self.F[t + ".norm3"] = ops.fold_layernorm(W[t + ".ff.net.0.proj.weight"], W[t + ".ff.net.0.proj.bias"],
                                                          W[t + ".norm3.weight"], W[t + ".norm3.bias"], geglu=True)
            elif k.endswith(".ff_norm.weight"):
                t = k[:-len(".ff_norm.weight")]
                self.F[t + ".ff_norm"] = ops.fold_layernorm(W[t + ".ff.net.0.proj.weight"], W[t + ".ff.net.0.proj.bias"],
                                                            W[t + ".ff_norm.weight"], W[t + ".ff_norm.bias"], geglu=True)
                for i in (0, 1):
                    a_ = f"{t}.attention_blocks.{i}"
                    self.F[f"{t}.norms.{i}"] = ops.fold_layernorm(W[a_ + ".qkv"], None, W[f"{t}.norms.{i}.weight"],
                                                                  W[f"{t}.norms.{i}.bias"])
                    # (LayerNorm(x) + pe) W^T = LayerNorm(x) W^T + pe W^T: the positional encoding becomes a per-frame bias
                    self._pe_proj[a_] = (W[a_ + ".pos_encoder.pe"] @ W[a_ + ".qkv"].float().t()).contiguous()

    def set_fp8(self, on: bool):
        """FP8 mode on / off; the e4m3 weights (ops.quantize_fp8_weight of the packed bf16 ones) are made on first use."""
        if on:
            _check_fp8_env()
            if not self.W8:
                # per output channel, so the packed q|k|v and GEGLU (value | gate) orders carry over to codes and scales
                self.W8 = {k: ops.quantize_fp8_weight(v) for k, v in self.W.items() if k.endswith(_FP8_KEYS)}
        self.fp8 = bool(on)

    def _gemm_p(self, a, w, bias, **kw):
        """A Linear whose output feeds a LayerNorm: (out, hand-over) -- the hand-over is the (parts, nparts) of
        ops.gemm_rowsums under the statistics hand-over, else None."""
        if self.ln_fuse:
            out, parts, n = ops.gemm_rowsums(a, w, bias, **kw)
            return out, (parts, n)
        return ops.gemm(a, w, bias, **kw), None

    def _ln_gemm(self, h, norm_key, w_key, *, geglu=False, pe=None, rows_per_frame=0, b=1, rs=None):
        """LayerNorm(h) [+ pe] -> Linear.  Default: the LayerNorm kernel followed by the GEMM.  With the producer's row sums
        `rs` (VX_LN_FUSE=1): one GEMM with the normalising epilogue; VX_LN_FOLD=1: statistics kernel + GEMM with the
        normalising epilogue.  FP8 mode: the LayerNorm writes e4m3 codes + row scales, the GEMM runs on e4m3 operands."""
        W = self.W
        if self.fp8:
            a8, a_scale = ops.layernorm_fp8(h, W[norm_key + ".weight"], W[norm_key + ".bias"], pe=pe,
                                            rows_per_frame=rows_per_frame)
            if geglu:
                w8, w_scale = self.W8[w_key + ".geglu_w"]
                return ops.gemm_fp8(a8, a_scale, w8, w_scale, W[w_key + ".geglu_b"], geglu=True)
            w8, w_scale = self.W8[w_key]
            return ops.gemm_fp8(a8, a_scale, w8, w_scale)
        if rs is None and not self.ln_fold:
            n = ops.layernorm(h, W[norm_key + ".weight"], W[norm_key + ".bias"], pe=pe, rows_per_frame=rows_per_frame)
            if geglu:
                return ops.gemm(n, W[w_key + ".geglu_w"], W[w_key + ".geglu_b"], geglu=True)
            return ops.gemm(n, W[w_key])
        wf, cs, bf = self.F[norm_key]
        bias2, div = None, 1
        if pe is not None:
            f = pe.shape[0]
            a_ = w_key[:-len(".qkv")]
            key = (a_, b, f)
            bias2 = self._pe_bias.get(key)
            if bias2 is None:
                bias2 = self._pe_proj[a_][:f].repeat(b, 1).contiguous()
                self._pe_bias[key] = bias2
            div = rows_per_frame
        if rs is not None:
            return ops.gemm_lnparts(h, wf, rs[0], rs[1], cs, bf, 1e-5, bias2=bias2, bias2_div=div, geglu=geglu)
        return ops.gemm_lnfold(h, wf, ops.row_stats(h), cs, bf, bias2=bias2, bias2_div=div, geglu=geglu)

    # ---------------------------------------------------------------- banks
    def _bank_kv(self, name: str, block: TemporalBasicTransformerBlock):
        """K/V of attn1_5 projected once per bank tensor (the reference re-projects f x steps x windows times,
        modules/mutual_self_attention.py:205-219).  The projected buffer is persistent per block and refreshed in
        place when the bank changes, so CUDA graphs that captured its address stay valid across videos."""
        if not block.bank:
            raise RuntimeError(f"{name}: reference bank is empty -- call ReferenceAttentionControl.update() first")
        bank = block.bank[0]
        key = (bank.data_ptr(), bank._version, tuple(bank.shape))
        hit = self._bank_cache.get(name)
        if hit is not None and hit[0] == key:
            return hit[1]
        bflat = bank.to(device=self.dev, dtype=BF16).reshape(-1, bank.shape[-1]).contiguous()
        w = self.W[name + ".attn1_5.kv"]
        buf = self._bank_buf.get(name)
        if buf is None or buf.shape != (bflat.shape[0], w.shape[0]):
            buf = torch.empty((bflat.shape[0], w.shape[0]), device=self.dev, dtype=BF16)
            self._bank_buf[name] = buf
            self.bank_epoch += 1
        ops.gemm(bflat, w, out=buf)
        # CFG: the uncond half of the bank is all zeros (reference mutual_self_attention.py:359) -> K = V = 0 ->
        # softmax-uniform x 0: the attention output of those frames is exactly 0, so it is not computed
        uncond_zero = bool(bank.shape[0] == 2 and torch.count_nonzero(bank[0]).item() == 0)
        if self._bank_flag.get(name) != uncond_zero:
            self._bank_flag[name] = uncond_zero
            self.bank_epoch += 1
        self._bank_cache[name] = (key, (buf, uncond_zero))
        return buf, uncond_zero

    def graph_signature(self):
        """Changes whenever a CUDA graph captured from forward_frames would be stale."""
        return (id(self), self.bank_epoch, self.fp8)

    # ---------------------------------------------------------------- blocks
    def _groupnorm(self, x, NB, HW, gamma, beta, eps, silu, x2=None, n=1):
        """ops.groupnorm in n launches of NB // n frames, the frame count of a one-sample forward.  The GroupNorm kernels
        pick their per-frame split (pixel chunks or cluster size, and with it the order in which partial statistics merge)
        from the number of frames in the launch; GroupNorm is per frame, so launches of one sample's frame count keep
        every frame's bits those of a one-sample forward."""
        if n == 1:
            return ops.groupnorm(x, NB, HW, gamma, beta, eps, silu, x2=x2, groups=self.groups)
        nb = NB // n
        out = torch.empty((NB * HW, x.shape[1] + (0 if x2 is None else x2.shape[1])), device=x.device, dtype=BF16)
        for s in range(n):
            r = slice(s * nb * HW, (s + 1) * nb * HW)
            ops.groupnorm(x[r], nb, HW, gamma, beta, eps, silu, x2=None if x2 is None else x2[r], groups=self.groups,
                          out=out[r])
        return out

    def _resnet(self, p, x, x2, NB, H, Wd, temb, n=1):
        W = self.W
        HW = H * Wd
        h = self._groupnorm(x, NB, HW, W[p + ".norm1.weight"], W[p + ".norm1.bias"], self.eps, True, x2=x2, n=n)
        off, co = self.temb_off[p + ".time_emb_proj"]
        h = ops.conv3x3(h.view(NB, H, Wd, -1), W[p + ".conv1.weight"], W[p + ".conv1.bias"],
                        bias2=temb[:, off:off + co], bias2_div=NB * HW)
        h = self._groupnorm(h, NB, HW, W[p + ".norm2.weight"], W[p + ".norm2.bias"], self.eps, True, n=n)
        if (p + ".conv_shortcut.weight") in W:
            sc = ops.gemm(x, W[p + ".conv_shortcut.weight"], W[p + ".conv_shortcut.bias"], a2=x2)
        else:
            assert x2 is None
            sc = x
        return ops.conv3x3(h.view(NB, H, Wd, -1), W[p + ".conv2.weight"], W[p + ".conv2.bias"], residual=sc)

    def _ff(self, p, n, res):
        W = self.W
        g = ops.gemm(n, W[p + ".net.0.proj.geglu_w"], W[p + ".net.0.proj.geglu_b"], geglu=True)   # GEGLU in the epilogue
        return ops.gemm(g, W[p + ".net.2.weight"], W[p + ".net.2.bias"], residual=res)

    def _spatial(self, p, x, NB, HW, f, enc_flat, n=1):
        W = self.W
        C = x.shape[1]
        heads = self.heads
        m = self.model
        h = self._groupnorm(x, NB, HW, W[p + ".norm.weight"], W[p + ".norm.bias"], 1e-6, False, n=n)
        h, rs = self._gemm_p(h, W[p + ".proj_in.weight"], W[p + ".proj_in.bias"])
        t = p + ".transformer_blocks.0"
        block = m.get_submodule(t)
        # attn1: self-attention
        qkv = self._ln_gemm(h, t + ".norm1", t + ".attn1.qkv", rs=rs)
        a = ops.flash_attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], heads, HW, HW)
        h, rs = self._gemm_p(a, W[t + ".attn1.to_out.0.weight"], W[t + ".attn1.to_out.0.bias"], residual=h)
        # attn1_5: reference attention, K/V from the bank: one K/V block per CFG half, shared by that half's n samples x f
        # frames (the batch is [uncond s0..s(n-1) | cond s0..s(n-1)]), so the bank holds NB // (n f) blocks of Nk rows
        q = self._ln_gemm(h, t + ".norm1_5", t + ".attn1_5.to_q.weight", rs=rs)
        kv, uncond_zero = self._bank_kv(t, block)
        nf = n * f
        Nk = kv.shape[0] // (NB // nf)
        if uncond_zero and NB == 2 * nf:
            a = torch.empty((NB * HW, C), device=self.dev, dtype=BF16)
            a[:nf * HW].zero_()
            ops.flash_attention(q[nf * HW:], kv[Nk:, :C], kv[Nk:, C:], heads, HW, Nk, kv_div=nf, out=a[nf * HW:])
        else:
            a = ops.flash_attention(q, kv[:, :C], kv[:, C:], heads, HW, Nk, kv_div=nf)
        h, rs = self._gemm_p(a, W[t + ".attn1_5.to_out.0.weight"], W[t + ".attn1_5.to_out.0.bias"],
                             scale=float(m.reference_attention_weight), residual=h)
        # attn2: audio cross-attention (5 tokens per frame)
        q = self._ln_gemm(h, t + ".norm2", t + ".attn2.to_q.weight", rs=rs)
        kv2 = ops.gemm(enc_flat, W[t + ".attn2.kv"])
        Lk = enc_flat.shape[0] // NB
        a = ops.smallkv_attention(q, kv2[:, :C], kv2[:, C:], HW, heads, Lk)
        h, rs = self._gemm_p(a, W[t + ".attn2.to_out.0.weight"], W[t + ".attn2.to_out.0.bias"],
                             scale=float(m.audio_attention_weight), residual=h)
        # feed-forward (GEGLU in the epilogue of the first GEMM)
        g = self._ln_gemm(h, t + ".norm3", t + ".ff.net.0.proj", geglu=True, rs=rs)
        h = ops.gemm(g, W[t + ".ff.net.2.weight"], W[t + ".ff.net.2.bias"], residual=h)
        return ops.gemm(h, W[p + ".proj_out.weight"], W[p + ".proj_out.bias"], residual=x)

    def _motion(self, p, x, NB, HW, b, f, n=1):
        """b: clips of f frames in the batch (all samples and CFG halves); n: samples (GroupNorm launch split)."""
        W = self.W
        p = p + ".temporal_transformer"
        C = x.shape[1]
        h = self._groupnorm(x, NB, HW, W[p + ".norm.weight"], W[p + ".norm.bias"], 1e-6, False, n=n)
        h, rs = self._gemm_p(h, W[p + ".proj_in.weight"], W[p + ".proj_in.bias"])
        t = p + ".transformer_blocks.0"
        for i in (0, 1):
            a_ = f"{t}.attention_blocks.{i}"
            pe = W[a_ + ".pos_encoder.pe"]
            if f > pe.shape[0]:
                raise ValueError(f"window of {f} frames exceeds temporal_position_encoding_max_len={pe.shape[0]}")
            qkv = self._ln_gemm(h, f"{t}.norms.{i}", a_ + ".qkv", pe=pe[:f], rows_per_frame=HW, b=b, rs=rs)
            a = ops.temporal_attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], b, f, HW, self.heads)
            h, rs = self._gemm_p(a, W[a_ + ".to_out.0.weight"], W[a_ + ".to_out.0.bias"], residual=h)
        g = self._ln_gemm(h, t + ".ff_norm", t + ".ff.net.0.proj", geglu=True, rs=rs)
        h = ops.gemm(g, W[t + ".ff.net.2.weight"], W[t + ".ff.net.2.bias"], residual=h)
        return ops.gemm(h, W[p + ".proj_out.weight"], W[p + ".proj_out.bias"], residual=x)

    # ---------------------------------------------------------------- forward
    def time_embedding(self, timestep) -> torch.Tensor:
        """[1, sum(Cout)] fp32: SiLU(time_embedding(t)) through all 22 time_emb_proj (unet_3d.py:449-470,
        resnet.py:225-228).  The timestep is a scalar broadcast to the batch, so one row serves all frames."""
        W = self.W
        if torch.is_tensor(timestep):
            t = timestep.detach().reshape(-1)[:1].to(device=self.dev, dtype=torch.float32)
        else:
            t = torch.tensor([float(timestep)], device=self.dev, dtype=torch.float32)
        e = ops.timestep_embed(t, self.boc[0])
        e = ops.skinny_linear(e, W["time_embedding.linear_1.weight"], W["time_embedding.linear_1.bias"], act_out=True)
        e = ops.skinny_linear(e, W["time_embedding.linear_2.weight"], W["time_embedding.linear_2.bias"])
        return ops.skinny_linear(e, W["temb_cat.weight"], W["temb_cat.bias"], act_in=True)

    def forward_frames(self, frames, timestep, enc, kps_nhwc, kps_frame_idx, b, f, temb=None, taps=None, n=1):
        """frames ((b n f),4,h,w) bf16; enc ((b n f),Lk,768); kps_nhwc [(frames) h w, C0] bf16 (rows gathered through
        kps_frame_idx when given).  Returns ((b n f),4,h,w) bf16.

        b is the CFG batch (2: uncond | cond, 1 without guidance) and n the number of samples of the same window: the batch
        is [uncond s0..s(n-1) | cond s0..s(n-1)], f frames per block.  Every launch whose schedule depends on the batch is
        split or shaped so that sample s comes out bit-identical to a one-sample forward of its blocks."""
        W = self.W
        NB, cin, H, Wd = frames.shape
        assert NB == b * n * f
        boc = self.boc
        if temb is None:
            temb = self.time_embedding(timestep)
        enc_flat = enc.to(BF16).reshape(-1, enc.shape[-1]).contiguous()

        def tap(name, t, hh, ww):
            if taps is not None:
                taps[name] = t.view(NB, hh, ww, -1).permute(0, 3, 1, 2).float()

        x = ops.conv_in(frames, W["conv_in.weight"], W["conv_in.bias"], boc[0], addend=kps_nhwc, add_frame=kps_frame_idx)
        tap("conv_in", x, H, Wd)
        skips = [(x, H, Wd)]
        h_, w_ = H, Wd
        for i in range(4):
            p = f"down_blocks.{i}"
            for j in range(2):
                x = self._resnet(f"{p}.resnets.{j}", x, None, NB, h_, w_, temb, n)
                tap(f"{p}.resnets.{j}", x, h_, w_)
                if i < 3:
                    x = self._spatial(f"{p}.attentions.{j}", x, NB, h_ * w_, f, enc_flat, n)
                    tap(f"{p}.attentions.{j}", x, h_, w_)
                x = self._motion(f"{p}.motion_modules.{j}", x, NB, h_ * w_, b * n, f, n)
                tap(f"{p}.motion_modules.{j}", x, h_, w_)
                skips.append((x, h_, w_))
            if i < 3:
                x = ops.downsample_conv(x, NB, h_, w_, W[f"{p}.downsamplers.0.conv.weight"], W[f"{p}.downsamplers.0.conv.bias"])
                h_, w_ = h_ // 2, w_ // 2
                tap(f"{p}.downsamplers.0", x, h_, w_)
                skips.append((x, h_, w_))
        x = self._resnet("mid_block.resnets.0", x, None, NB, h_, w_, temb, n)
        x = self._spatial("mid_block.attentions.0", x, NB, h_ * w_, f, enc_flat, n)
        x = self._motion("mid_block.motion_modules.0", x, NB, h_ * w_, b * n, f, n)
        x = self._resnet("mid_block.resnets.1", x, None, NB, h_, w_, temb, n)
        tap("mid_block", x, h_, w_)
        for i in range(4):
            p = f"up_blocks.{i}"
            for j in range(3):
                skip, sh, sw = skips.pop()
                assert (sh, sw) == (h_, w_)
                x = self._resnet(f"{p}.resnets.{j}", x, skip, NB, h_, w_, temb, n)
                tap(f"{p}.resnets.{j}", x, h_, w_)
                if i > 0:
                    x = self._spatial(f"{p}.attentions.{j}", x, NB, h_ * w_, f, enc_flat, n)
                    tap(f"{p}.attentions.{j}", x, h_, w_)
                x = self._motion(f"{p}.motion_modules.{j}", x, NB, h_ * w_, b * n, f, n)
                tap(f"{p}.motion_modules.{j}", x, h_, w_)
            if i < 3:
                # Upsample3D (modules/resnet.py:53-90): nearest x2 + conv3x3, without the 4x intermediate
                x = ops.upconv3x3(x.view(NB, h_, w_, -1), W[f"{p}.upsamplers.0.conv.weight"], W[f"{p}.upsamplers.0.conv.bias"])
                h_, w_ = 2 * h_, 2 * w_
                tap(f"{p}.upsamplers.0", x, h_, w_)
        x = self._groupnorm(x, NB, h_ * w_, W["conv_norm_out.weight"], W["conv_norm_out.bias"], self.eps, True, n=n)
        out = torch.empty((NB, self.model.config["out_channels"], H, Wd), device=self.dev, dtype=BF16)
        ops.conv_out_tc(x, NB, H, Wd, W["conv_out.packed_w"], W["conv_out.packed_b"], out)
        return out
