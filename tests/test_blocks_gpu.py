"""The engine's blocks (UNet, ReferenceNet, VAE) against their fp64 oracle blocks, teacher-forced, one residual branch
at a time.

The kernel bound tests check each kernel; this file checks how ``UNetEngine`` / ``RefNetEngine`` / the VAE engines put
them together: which bank block a frame attends to, which audio tokens and positional-encoding row a frame gets, which
time-embedding slice a resnet reads, the skip-concat order, and where the reference and audio weights apply.  Whole-
network relative-L2 checks cannot see such errors: the residual stream dominates every tap.  So each case

1. builds the block from a synthetic state dict (``O.synth_state_dict``) in which the output projections (weight and
   bias) of every branch but one are zeroed -- attn1, attn1_5, attn2, ff.net.2 of a spatial transformer; the two
   attention blocks' to_out and ff.net.2 of a motion module; conv2 of a resnet -- and the tested branch may be scaled
   (``SPATIAL_GAIN``, ``MOTION_GAIN``, ``WRITE_GAIN``) until it carries at least half of the block's change ``||ref64 - x||`` (asserted on the fp64 data);
2. runs one engine block method on a bf16 input;
3. runs the oracle block in fp64 on exactly that input with the bf16-rounded weights (``ref64``), and again with the
   tested branch zeroed too: the branch is ``B = ref64 - ref64(B zeroed)``;
4. runs the oracle block in torch.bfloat16 on the CPU: the reference's own eager arithmetic, the yardstick.

Criterion: ``e_prod = ||out - ref64|| / ||B||`` and ``e_eager`` the same measure of the bf16 CPU run;
``e_prod <= min(max(1.5 e_eager, FLOOR), CEIL)``, and no NaN / Inf.  Blocks without a residual (time embedding, conv_in,
down / up sampling convs, conv_out, VAE decode, the ReferenceNet bank) use B = the whole output.

Fault catalogue (``test_fault_catalogue``, CPU only): each fault is emulated in the fp64 oracle at the case where the
engine could make it, and must move that case's measure by at least 2x its threshold.  Fault size / threshold, CPU:

    pe rows shifted by one frame          1.65e-1 / 1.02e-2     audio tokens of the neighbouring frame   1.40   / 1.00e-2
    two clips in one temporal attention   4.32e-1 / 1.02e-2     uncond-zero shortcut without the bias    1.10e-1 / 1.02e-2
    reference weight applied as 1.0       5.26e-2 / 1.02e-2     time embedding of the neighbouring slice 1.39   / 1.00e-2
    reference weight on the residual too  4.14e-2 / 1.02e-2     time embedding without its SiLU          9.82e-1 / 1.00e-2
    audio weight off by 3 %               3.00e-2 / 1.00e-2     skip and x concatenated the other way    4.08   / 1.27e-2
    CFG bank halves swapped               1.14    / 1.00e-2     GroupNorm statistics over all frames     4.74e-1 / 1.14e-2
    sample s reads s+1's bank (kv_div f)  6.15e-1 / 1.00e-2
No listed fault is invisible; the smallest ratio is 3.0 (audio weight: the branch is isolated, so 3 % of it is 3e-2).

Thresholds.  FLOOR = 1e-2 and CEIL = 1.45e-2 sit below half the smallest fault (3.0e-2).  They rest on these measured
values (e_eager on the CPU; e_prod on an H100 80GB HBM3 at its 700 W power limit):
    spatial transformer, 4 branches x 5 batch forms x f 4, 24, small widths and head dims 40 / 80 / 160:
        e_eager 5.6e-3 - 8.7e-3, e_prod 4.7e-3 - 7.9e-3 (at most 0.62 of the threshold), branch share 0.65 - 0.94
    motion module, 3 branches x f 1, 2, 16, 17, 24, 32 x b.n 1, 2, 4: e_eager 4.8e-3 - 8.1e-3, e_prod 3.9e-3 - 6.0e-3
    resnets: e_eager 7.1e-3 - 8.5e-3, e_prod 5.6e-3 - 7.4e-3;  time embedding (fp32 in the engine): e_eager 3.3e-3 -
        5.2e-3, e_prod <= 1.7e-3;  convs without residual (conv_in, down / up sampling, conv_out): e_eager 1.7e-3 -
        3.1e-3, e_prod 1.7e-3 - 2.4e-3 (the up-sampling convs, 1.4x e_eager, use weights summed per output parity and
        rounded to bf16 once more);  ReferenceNet write block and bank: e_eager 2.9e-3 - 8.6e-3, e_prod 2.9e-3 - 7.9e-3
    VAE: the mid attention (single head over 64 tokens: its output averages values, the error does not) and the whole
        decode are the largest: e_eager 1.43e-2 / 1.42e-2, e_prod 1.37e-2 / 1.26e-2 -- what sets CEIL.
FLOOR keeps a case whose eager run is unusually accurate from a threshold tighter than storing its output in bf16.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import vx_oracle as O
from test_unet_gpu import UNET_EXTRA

BF16 = torch.bfloat16
F64 = torch.float64
CFG = O.small_cfg()
HEADS, GROUPS, EPS = 8, 32, 1e-5
REF_W, AUDIO_W = 0.95, 3.0
FLOOR, CEIL = 1e-2, 1.45e-2
MIN_SHARE = 0.5

SPATIAL_BRANCHES = {"attn1": "attn1.to_out.0", "attn1_5": "attn1_5.to_out.0", "attn2": "attn2.to_out.0",
                    "ff": "ff.net.2"}
MOTION_BRANCHES = {"attn0": "attention_blocks.0.to_out.0", "attn1": "attention_blocks.1.to_out.0", "ff": "ff.net.2"}
WRITE_BRANCHES = {"attn1": "attn1.to_out.0", "attn2": "attn2.to_out.0", "ff": "ff.net.2"}
# Gains of the tested branch's output projection (powers of two: exact in bf16), so that it carries at least half of the
# block's change.  Measured shares at gain 1 (fp64, f = 4, small and full width): spatial attn1 0.21-0.36, attn1_5
# 0.14-0.34 (its bank rows are LayerNorm outputs; the proj_in pass-through dominates), attn2 0.86-0.87, ff 0.54-0.56;
# motion attention blocks 0.53-0.78 (falling with f), ff 0.55; ReferenceNet write block as the spatial one.
SPATIAL_GAIN = {"attn1": 4.0, "attn1_5": 8.0, "ff": 2.0}
MOTION_GAIN = {"attn0": 2.0, "attn1": 2.0, "ff": 2.0}
WRITE_GAIN = {"attn1": 4.0, "ff": 2.0}

# batch forms of the spatial transformer: (b, n, uncond bank half)
FORMS = {"zero-uncond": (2, 1, "zero"),       # the CFG shortcut: uncond attention output is to_out's bias
         "uncond": (2, 1, "rand"),            # non-zero uncond bank: the general path
         "b1": (1, 1, None),
         "n2": (2, 2, "zero"),                # two samples, [u s0, u s1 | c s0, c s1]
         "n2-uncond": (2, 2, "rand")}
SPATIAL_LEVELS = {0: ("down_blocks.0.attentions.0", 8), 1: ("down_blocks.1.attentions.0", 8),
                  2: ("down_blocks.2.attentions.0", 4)}
FULL_LEVELS = {40: ("down_blocks.0.attentions.0", 8), 80: ("down_blocks.1.attentions.0", 4),
               160: ("down_blocks.2.attentions.0", 4)}
MOTION_BLOCK, MOTION_H = "down_blocks.1.motion_modules.0", 4
RESNETS = {"down": ("down_blocks.1.resnets.0", 8, None),            # 64 -> 128, conv_shortcut
           "mid": ("mid_block.resnets.0", 4, None),
           "up": ("up_blocks.1.resnets.0", 4, True)}    # [x 256 | skip 256] -> 256, conv_shortcut
RESULTS = []


# ------------------------------------------------------------------------------------------------------------ helpers
def _seed(*xs):
    s = 0
    for v in xs:
        s = (s * 1000003 + sum(map(ord, str(v)))) % (1 << 31)
    return s


def _gen(*xs):
    return torch.Generator().manual_seed(_seed(*xs))


def _frames(g, B, C, H, W):
    """bf16 activations whose frames differ in scale and offset (per-frame statistics that a GroupNorm over the wrong
    frames would mix)."""
    s = 0.5 + 1.5 * torch.rand(B, 1, 1, 1, generator=g)
    m = 2 * torch.rand(B, 1, 1, 1, generator=g) - 1
    return (torch.randn(B, C, H, W, generator=g) * s + m).to(BF16)


def _ln_rows(t):
    return O._ln_rows(t).to(BF16)


def _sub(sd, *prefixes):
    return {k: v for k, v in sd.items() if k.startswith(prefixes)}


def _cast(sd, dtype):
    """Weights rounded to bf16 (what ``.to(bfloat16)`` does to the model), then held in ``dtype``."""
    return {k: v.to(BF16).to(dtype) for k, v in sd.items()}


def isolate(sd, tb, branches, keep, gain=1.0, drop_keep=False):
    """Zero the output projections (weight and bias) of every branch but ``keep``, scale ``keep``'s by ``gain``, or
    zero it too (``drop_keep``)."""
    out = dict(sd)
    for name, key in branches.items():
        s = 0.0 if (name != keep or drop_keep) else gain
        if s != 1.0:
            for leaf in ("weight", "bias"):
                out[f"{tb}.{key}.{leaf}"] = sd[f"{tb}.{key}.{leaf}"] * s
    return out


def _norm(t):
    return float(t.double().norm())


def _measure(out, ref, B):
    return _norm(out.double() - ref) / max(_norm(B), 1e-30)


def threshold(e_eager):
    return min(max(1.5 * e_eager, FLOOR), CEIL)


def _tok(x):
    """(B, C, H, W) -> [(B H W), C] bf16 on the device (cast on the host)."""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).to(BF16).contiguous().cuda()


def _img(t, B, H, W):
    return t.float().cpu().view(B, H, W, -1).permute(0, 3, 1, 2).double()


def judge(name, out, c):
    """Record one case and return its failure message ('' when it passes)."""
    out = out.double()
    e_prod = _measure(out, c["ref"], c["B"])
    thr = threshold(c["e_eager"])
    finite = bool(torch.isfinite(out).all())
    RESULTS.append((name, e_prod, c["e_eager"], c.get("share", float("nan")), thr))
    print(f"{name:58s} e_prod {e_prod:.3e}  e_eager {c['e_eager']:.3e}  share {c.get('share', float('nan')):.2f}  "
          f"thr {thr:.2e}")
    if not finite:
        return f"{name}: NaN / Inf in the output"
    if not e_prod <= thr:
        return f"{name}: e_prod {e_prod:.3e} > threshold {thr:.3e} (e_eager {c['e_eager']:.3e})"
    return ""


def _finish(c, ref, zero, eager, x_res=None):
    """Attach B, the share of the block delta it carries, and e_eager to case ``c``."""
    c["ref"] = ref
    c["B"] = ref - zero if zero is not None else ref
    if x_res is not None:
        c["share"] = _norm(c["B"]) / max(_norm(ref - x_res), 1e-30)
    c["e_eager"] = _measure(eager, ref, c["B"])
    return c


# ----------------------------------------------------------------------------------------------- spatial transformer
def spatial_inputs(C, H, form, f, seed):
    b, n, unc = FORMS[form]
    B = b * n * f
    g = _gen("spatial", C, H, form, f, seed)
    x = _frames(g, B, C, H, H)
    enc = _ln_rows(torch.randn(B, 5, CFG["cross_attention_dim"], generator=g))
    cond = _ln_rows(torch.randn(1, H * H, C, generator=g))
    if b == 1:
        bank = cond
    else:
        bank = torch.cat([torch.zeros_like(cond) if unc == "zero" else _ln_rows(torch.randn(1, H * H, C, generator=g)),
                          cond])
    return dict(x=x, enc=enc, bank=bank, b=b, n=n, f=f, form=form)


def spatial_ref(sd, p, c, dtype, ref_w=REF_W, audio_w=AUDIO_W, bank_clips=None, enc=None):
    """O.spatial_transformer on case ``c``: clip k (f frames) reads bank block k // n."""
    bank = c["bank"].to(dtype)
    if bank_clips is None:
        bank_clips = bank.repeat_interleave(c["n"], 0)
    enc = c["enc"] if enc is None else enc
    with torch.no_grad():
        return O.spatial_transformer(sd, p, c["x"].to(dtype), enc.to(dtype), bank_clips.to(dtype), HEADS, GROUPS,
                                     ref_w, audio_w, c["f"])


def spatial_case(sd, p, branch, form, f, H, seed=0):
    """fp64 / bf16 oracle data of one isolated-branch spatial case on the full state dict ``sd``."""
    tb = p + ".transformer_blocks.0"
    sub = _sub(sd, p + ".")
    C = sub[p + ".norm.weight"].shape[0]
    iso = isolate(sub, tb, SPATIAL_BRANCHES, branch, SPATIAL_GAIN.get(branch, 1.0))
    c = spatial_inputs(C, H, form, f, seed)
    sd64 = _cast(iso, F64)
    c["sd64"], c["sd_zero64"] = sd64, _cast(isolate(sub, tb, SPATIAL_BRANCHES, branch, drop_keep=True), F64)
    c["iso"], c["p"] = iso, p
    ref = spatial_ref(sd64, p, c, F64)
    zero = spatial_ref(c["sd_zero64"], p, c, F64)
    eager = spatial_ref(_cast(iso, BF16), p, c, BF16).double()
    return _finish(c, ref, zero, eager, x_res=c["x"].double())


def run_spatial(model, c, keep):
    eng = model.engine()
    p = c["p"]
    bank = c["bank"].cuda()
    keep.append(bank)   # the bank K/V cache is keyed by address: a freed bank must not lend its address to the next one
    model.get_submodule(p + ".transformer_blocks.0").bank = [bank]
    model.reference_attention_weight, model.audio_attention_weight = REF_W, AUDIO_W
    B, C, H, W = c["x"].shape
    enc = c["enc"].reshape(-1, c["enc"].shape[-1]).contiguous().cuda()
    y = eng._spatial(p, _tok(c["x"]), B, H * W, c["f"], enc, c["n"])
    torch.cuda.synchronize()
    return _img(y, B, H, W)


# ---------------------------------------------------------------------------------------------------- motion module
def motion_case(sd, p, branch, bn, f, H=MOTION_H, seed=0, pe=None):
    tb = p + ".temporal_transformer.transformer_blocks.0"
    sub = _sub(sd, p + ".")
    C = sub[p + ".temporal_transformer.norm.weight"].shape[0]
    iso = isolate(sub, tb, MOTION_BRANCHES, branch, MOTION_GAIN.get(branch, 1.0))
    x = _frames(_gen("motion", C, H, bn, f, seed), bn * f, C, H, H)
    c = dict(x=x, f=f, bn=bn, p=p, iso=iso)
    c["sd64"] = _cast(iso, F64)
    with torch.no_grad():
        ref = O.motion_module(c["sd64"], p, x.double(), HEADS, GROUPS, f)
        zero = O.motion_module(_cast(isolate(sub, tb, MOTION_BRANCHES, branch, drop_keep=True), F64), p, x.double(),
                               HEADS, GROUPS, f)
        eager = O.motion_module(_cast(iso, BF16), p, x, HEADS, GROUPS, f).double()
    return _finish(c, ref, zero, eager, x_res=x.double())


def _motion_split(bn):
    """b . n clips as (clips, samples): 4 clips are two CFG halves of two samples."""
    return bn, (2 if bn == 4 else 1)


def run_motion(model, c):
    B, C, H, W = c["x"].shape
    clips, n = _motion_split(c["bn"])
    y = model.engine()._motion(c["p"], _tok(c["x"]), B, H * W, clips, c["f"], n)
    torch.cuda.synchronize()
    return _img(y, B, H, W)


# ----------------------------------------------------------------------------------------------------------- resnets
def temb_chain(sd, t, dtype):
    """``emb`` of the reference (unet_3d.py:449-470): linear_2(SiLU(linear_1(sinusoid(t)))), one row."""
    e = O.timestep_embedding(torch.tensor([float(t)]), CFG["block_out_channels"][0]).to(dtype)
    return O._lin(sd, "time_embedding.linear_2", F.silu(O._lin(sd, "time_embedding.linear_1", e)))


def resnet_case(sd, kind, n, f=4, t=499, seed=0, skip_first=False):
    p, H, has_skip = RESNETS[kind]
    sub = _sub(sd, p + ".", "time_embedding.")
    ci = sub[p + ".norm1.weight"].shape[0]
    B = 2 * n * f
    g = _gen("resnet", kind, n, f, seed)
    if not has_skip:
        x, x2 = _frames(g, B, ci, H, H), None
    else:
        x, x2 = _frames(g, B, ci // 2, H, H), _frames(g, B, ci // 2, H, H)
    iso = isolate(sub, p, {"conv2": "conv2"}, "conv2")
    c = dict(x=x, x2=x2, n=n, p=p, t=t, iso=iso, H=H)

    def run(sd_, dtype):
        xin = x.to(dtype) if x2 is None else torch.cat([x2, x] if skip_first else [x, x2], 1).to(dtype)
        emb = temb_chain(sd_, t, dtype).expand(B, -1)
        with torch.no_grad():
            return O.resnet_block(sd_, p, xin, emb, GROUPS, EPS)
    c["run"] = run
    sd64 = _cast(iso, F64)
    c["sd64"] = sd64
    ref = run(sd64, F64)
    zero = run(_cast(isolate(sub, p, {"conv2": "conv2"}, "conv2", drop_keep=True), F64), F64)
    eager = run(_cast(iso, BF16), BF16).double()
    # with a conv_shortcut, B is the whole residual branch by construction (the rest is the shortcut of x)
    return _finish(c, ref, zero, eager, x_res=x.double() if x2 is None and ref.shape == x.shape else None)


# ------------------------------------------------------------------------------------------------------ state dicts
_SD = {}


def small_sd():
    if "unet" not in _SD:
        _SD["unet"] = O.synth_state_dict(O.unet_param_shapes(CFG), 4321)
    return _SD["unet"]


def _full_keys(prefixes):
    shapes = O.unet_param_shapes(O.DEFAULT_CFG)
    return O.synth_state_dict({k: s for k, s in shapes.items() if k.startswith(prefixes)}, 4322)


# ====================================================================================================== CPU: faults
def _spatial_fault_case(branch, form, f=4):
    return spatial_case(small_sd(), SPATIAL_LEVELS[0][0], branch, form, f, SPATIAL_LEVELS[0][1])


def _fault_ref_weight_one():
    c = _spatial_fault_case("attn1_5", "zero-uncond")
    return c, spatial_ref(c["sd64"], c["p"], c, F64, ref_w=1.0)


def _fault_ref_weight_on_residual():
    # under isolation the block is x + proj_out(h0 + w a) (h0 = proj_in(GroupNorm(x))); applying w to the residual as
    # well, w (h0 + a), adds (w - 1) proj_out.weight h0 = (w - 1) (ref(attn1_5 zeroed) - x - proj_out.bias)
    c = _spatial_fault_case("attn1_5", "zero-uncond")
    zero = spatial_ref(c["sd_zero64"], c["p"], c, F64)
    bias = c["sd64"][c["p"] + ".proj_out.bias"].view(1, -1, 1, 1)
    return c, c["ref"] + (REF_W - 1) * (zero - c["x"].double() - bias)


def _fault_uncond_bias_dropped():
    # the shortcut writes zero attention for the uncond frames; their to_out must still add its bias (x weight)
    c = _spatial_fault_case("attn1_5", "zero-uncond")
    zero = spatial_ref(c["sd_zero64"], c["p"], c, F64)
    half = c["x"].shape[0] // 2
    return c, torch.cat([zero[:half], c["ref"][half:]])


def _fault_cfg_swapped():
    c = _spatial_fault_case("attn1_5", "uncond")
    return c, spatial_ref(c["sd64"], c["p"], c, F64, bank_clips=c["bank"].flip(0))


def _fault_kv_div_f():
    # kv_div = f instead of n f: clip k reads bank block k (u s1 reads the cond block; beyond the bank, the last block)
    c = _spatial_fault_case("attn1_5", "n2-uncond")
    bank = c["bank"]
    clips = torch.stack([bank[min(k, bank.shape[0] - 1)] for k in range(c["b"] * c["n"])])
    return c, spatial_ref(c["sd64"], c["p"], c, F64, bank_clips=clips)


def _fault_audio_weight():
    c = _spatial_fault_case("attn2", "zero-uncond")
    return c, spatial_ref(c["sd64"], c["p"], c, F64, audio_w=AUDIO_W * 0.97)


def _fault_audio_neighbour():
    c = _spatial_fault_case("attn2", "zero-uncond")
    return c, spatial_ref(c["sd64"], c["p"], c, F64, enc=c["enc"].roll(-1, 0))


def _motion_fault_case():
    return motion_case(small_sd(), MOTION_BLOCK, "attn0", 2, 16)


def _fault_pe_shift():
    c = _motion_fault_case()
    sd = dict(c["sd64"])
    k = c["p"] + ".temporal_transformer.transformer_blocks.0.attention_blocks.0.pos_encoder.pe"
    sd[k] = O.positional_encoding(sd[k].shape[2], sd[k].shape[1] + 1)[:, 1:].to(BF16).double()
    with torch.no_grad():
        return c, O.motion_module(sd, c["p"], c["x"].double(), HEADS, GROUPS, c["f"])


def _fault_two_clips():
    # the two clips attend as one sequence of 2f frames; each keeps its own positional-encoding rows
    c = _motion_fault_case()
    sd = dict(c["sd64"])
    for i in (0, 1):
        k = c["p"] + f".temporal_transformer.transformer_blocks.0.attention_blocks.{i}.pos_encoder.pe"
        sd[k] = sd[k][:, :c["f"]].repeat(1, 2, 1)
    with torch.no_grad():
        return c, O.motion_module(sd, c["p"], c["x"].double(), HEADS, GROUPS, 2 * c["f"])


def _temb_case(t=499):
    sd = _cast(_sub(small_sd(), "time_embedding.", "down_blocks.1.resnets."), F64)
    emb = temb_chain(sd, t, F64)
    p = "down_blocks.1.resnets.0.time_emb_proj"
    ref = O._lin(sd, p, F.silu(emb))
    sd16 = _cast(_sub(small_sd(), "time_embedding.", "down_blocks.1.resnets."), BF16)
    eager = O._lin(sd16, p, F.silu(temb_chain(sd16, t, BF16))).double()
    return _finish(dict(sd64=sd, emb=emb), ref, None, eager)


def _fault_temb_neighbour():
    c = _temb_case()
    return c, O._lin(c["sd64"], "down_blocks.1.resnets.1.time_emb_proj", F.silu(c["emb"]))


def _fault_temb_no_silu():
    c = _temb_case()
    return c, O._lin(c["sd64"], "down_blocks.1.resnets.0.time_emb_proj", c["emb"])


def _fault_skip_order():
    c = resnet_case(small_sd(), "up", 1)
    return c, resnet_case(small_sd(), "up", 1, skip_first=True)["ref"]


def _gn_all_frames(sd, p, x, groups, eps):
    B, C, H, W = x.shape
    y = F.group_norm(x.transpose(0, 1).reshape(1, C, B * H, W), groups, sd[p + ".weight"], sd[p + ".bias"], eps)
    return y.reshape(C, B, H, W).transpose(0, 1)


def _fault_gn_all_frames(monkeypatch):
    c = resnet_case(small_sd(), "down", 1)
    monkeypatch.setattr(O, "group_norm", _gn_all_frames)
    return c, c["run"](c["sd64"], F64)


FAULTS = {
    "pe-shifted-one-frame": _fault_pe_shift,
    "temporal-two-clips-grouped": _fault_two_clips,
    "ref-weight-as-1": _fault_ref_weight_one,
    "ref-weight-on-residual": _fault_ref_weight_on_residual,
    "audio-weight-3pct": _fault_audio_weight,
    "cfg-bank-halves-swapped": _fault_cfg_swapped,
    "bank-kv-div-f": _fault_kv_div_f,
    "audio-neighbour-frame": _fault_audio_neighbour,
    "uncond-shortcut-drops-bias": _fault_uncond_bias_dropped,
    "temb-neighbour-slice": _fault_temb_neighbour,
    "temb-missing-silu": _fault_temb_no_silu,
    "skip-concat-order": _fault_skip_order,
    "groupnorm-over-all-frames": _fault_gn_all_frames,
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_fault_catalogue(fault, monkeypatch):
    """Each fault, emulated in the fp64 oracle, moves its case's measure by at least twice the case's threshold."""
    fn = FAULTS[fault]
    c, bad = fn(monkeypatch) if fault == "groupnorm-over-all-frames" else fn()
    size = _measure(bad, c["ref"], c["B"])
    thr = threshold(c["e_eager"])
    print(f"{fault:28s} fault {size:.3e}  threshold {thr:.3e}  ratio {size / thr:.1f}  (e_eager {c['e_eager']:.3e})")
    assert size >= 2 * thr and size >= 2 * CEIL


def test_isolated_branches_dominate():
    """On the fp64 data every isolated branch carries at least half of its block's change (gains applied)."""
    sd = small_sd()
    for branch in SPATIAL_BRANCHES:
        for form in ("zero-uncond", "uncond"):
            c = spatial_case(sd, SPATIAL_LEVELS[1][0], branch, form, 4, SPATIAL_LEVELS[1][1])
            assert c["share"] >= MIN_SHARE, (branch, form, c["share"])
    for branch in MOTION_BRANCHES:
        c = motion_case(sd, MOTION_BLOCK, branch, 2, 4)
        assert c["share"] >= MIN_SHARE, (branch, c["share"])
    assert resnet_case(sd, "mid", 1)["share"] >= MIN_SHARE


def test_emulation_helpers_match_the_oracle():
    """The restated pieces the fault catalogue uses agree with the oracle where they must: the time-embedding chain
    with O.unet_forward's, GroupNorm over all frames with per-frame GroupNorm on one frame."""
    sd = _cast(_sub(small_sd(), "conv_norm_out.", "time_embedding."), F64)
    x = _frames(_gen("gn"), 1, 64, 4, 4).double()
    assert torch.allclose(_gn_all_frames(sd, "conv_norm_out", x, GROUPS, EPS),
                          O.group_norm(sd, "conv_norm_out", x, GROUPS, EPS), atol=1e-12)
    e = temb_chain(sd, 999, F64)
    t_emb = O.timestep_embedding(torch.tensor([999]), 64).double()
    assert torch.allclose(e, O._lin(sd, "time_embedding.linear_2", F.silu(O._lin(sd, "time_embedding.linear_1", t_emb))))


# ================================================================================================== GPU: the blocks
pytest_gpu = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _table():
    yield
    if RESULTS:
        print(f"\n{'case':58s} {'e_prod':>9s} {'e_eager':>9s} {'share':>6s} {'thr':>9s}")
        for name, ep, ee, sh, thr in RESULTS:
            print(f"{name:58s} {ep:9.3e} {ee:9.3e} {sh:6.2f} {thr:9.2e}")


def _unet(cfg, sd, full=False):
    from vexpress_b200.modules import UNet3DConditionModel
    kw = dict(block_out_channels=cfg["block_out_channels"], cross_attention_dim=cfg["cross_attention_dim"], **UNET_EXTRA)
    if full:
        # the full-width blocks under test get weights; the rest of the model stays uninitialised device memory
        with torch.device("cuda"):
            model = UNet3DConditionModel(**kw)
        model.load_state_dict(sd, strict=False)
    else:
        model = UNet3DConditionModel(**kw)
        model.load_state_dict(sd, strict=True)
    return model.to(BF16).to("cuda")


def _load(model, sd):
    """Copy the (isolated) block weights ``sd`` into the model; the engine is repacked on next use."""
    with torch.no_grad():
        for k, v in sd.items():
            if not k.endswith(".pe"):
                model.get_parameter(k).copy_(v)
    model._engine = None
    return model.engine()


@pytest.fixture(scope="module")
def small():
    from vexpress_b200 import _ffi
    _ffi.require_sm90()
    return _unet(CFG, small_sd())


@pytest.fixture(scope="module")
def full():
    prefixes = tuple(p + "." for p, _ in FULL_LEVELS.values())
    sd = _full_keys(prefixes)
    return sd, _unet(O.DEFAULT_CFG, sd, full=True)


def _spatial_sweep(model, sd, p, H, branch, forms, frames, tag):
    bad, keep = [], []
    _load(model, isolate(_sub(sd, p + "."), p + ".transformer_blocks.0", SPATIAL_BRANCHES, branch,
                         SPATIAL_GAIN.get(branch, 1.0)))
    for f in frames:
        for form in forms:
            c = spatial_case(sd, p, branch, form, f, H)
            assert c["share"] >= MIN_SHARE, (p, branch, form, c["share"])
            bad.append(judge(f"spatial {tag} {branch} {form} f={f}", run_spatial(model, c, keep), c))
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest_gpu
@pytest.mark.parametrize("branch", list(SPATIAL_BRANCHES))
@pytest.mark.parametrize("level", list(SPATIAL_LEVELS))
def test_spatial_transformer_branch(small, level, branch):
    p, H = SPATIAL_LEVELS[level]
    _spatial_sweep(small, small_sd(), p, H, branch, list(FORMS), (4, 24), f"L{level}")


@pytest_gpu
@pytest.mark.parametrize("branch", list(SPATIAL_BRANCHES))
@pytest.mark.parametrize("hd", list(FULL_LEVELS))
def test_spatial_transformer_fullwidth_branch(full, hd, branch):
    sd, model = full
    p, H = FULL_LEVELS[hd]
    _spatial_sweep(model, sd, p, H, branch, list(FORMS), (4,), f"hd{hd}")


@pytest_gpu
@pytest.mark.parametrize("f", [1, 2, 16, 17, 24, 32])
@pytest.mark.parametrize("branch", list(MOTION_BRANCHES))
def test_motion_module_branch(small, branch, f):
    sd = small_sd()
    p = MOTION_BLOCK
    _load(small, isolate(_sub(sd, p + "."), p + ".temporal_transformer.transformer_blocks.0", MOTION_BRANCHES, branch,
                         MOTION_GAIN.get(branch, 1.0)))
    bad = []
    for bn in (1, 2, 4):
        c = motion_case(sd, p, branch, bn, f)
        assert c["share"] >= MIN_SHARE, (branch, f, bn, c["share"])
        bad.append(judge(f"motion {branch} f={f} bn={bn}", run_motion(small, c), c))
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest_gpu
def test_motion_module_rejects_window_beyond_pe(small):
    eng = small.engine()
    C = CFG["block_out_channels"][1]
    x = torch.zeros((33 * 4, C), device="cuda", dtype=BF16)
    with pytest.raises(ValueError, match="exceeds temporal_position_encoding_max_len"):
        eng._motion(MOTION_BLOCK, x, 33, 4, 1, 33)


@pytest_gpu
@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("kind", list(RESNETS))
def test_resnet_branch(small, kind, n):
    sd = small_sd()
    c = resnet_case(sd, kind, n)
    assert c.get("share", 1.0) >= MIN_SHARE, (kind, c["share"])
    eng = _load(small, c["iso"])
    B, ci, H, W = c["x"].shape
    temb = eng.time_embedding(c["t"])
    x2 = None if c["x2"] is None else _tok(c["x2"])
    y = eng._resnet(c["p"], _tok(c["x"]), x2, B, H, W, temb, n)
    torch.cuda.synchronize()
    assert not judge(f"resnet {kind} n={n}", _img(y, B, H, W), c)


@pytest_gpu
@pytest.mark.parametrize("as_tensor", [False, True])
@pytest.mark.parametrize("t", [0, 1, 499, 999])
def test_time_embedding_slices(small, t, as_tensor):
    """time_embedding() sliced at every resnet's temb_off against SiLU -> that resnet's time_emb_proj of the chain."""
    sd = small_sd()
    eng = _load(small, _sub(sd, "time_embedding."))
    temb = eng.time_embedding(torch.tensor([t]).cuda() if as_tensor else t).double().cpu()
    temb_sd = {k: v for k, v in sd.items() if "time_emb" in k}
    sd64, sd16 = _cast(temb_sd, F64), _cast(temb_sd, BF16)
    emb64, emb16 = temb_chain(sd64, t, F64), temb_chain(sd16, t, BF16)
    bad = []
    assert len(eng.temb_off) == 22
    for key, (off, co) in eng.temb_off.items():
        c = _finish({}, O._lin(sd64, key, F.silu(emb64)), None, O._lin(sd16, key, F.silu(emb16)).double())
        bad.append(judge(f"temb t={t} {'tensor' if as_tensor else 'float'} {key[:-14]}", temb[:, off:off + co], c))
    assert not any(bad), "\n".join(b for b in bad if b)


def _plain_case(ref, eager, zero=None):
    return _finish({}, ref, zero, eager)


@pytest_gpu
@pytest.mark.parametrize("frame_idx", [False, True])
def test_conv_in_with_kps(small, frame_idx):
    from vexpress_b200 import ops
    sd = small_sd()
    eng = _load(small, _sub(sd, "conv_in."))
    g = _gen("conv_in", frame_idx)
    B, H, C0 = 8, 16, CFG["block_out_channels"][0]
    x = torch.randn(B, 4, H, H, generator=g).to(BF16)
    kps = (0.1 * torch.randn(B, C0, H, H, generator=g)).to(BF16)
    idx = torch.randperm(B, generator=g) if frame_idx else torch.arange(B)
    kps_rows = kps[idx].double()
    sd64, sd16 = _cast(_sub(sd, "conv_in."), F64), _cast(_sub(sd, "conv_in."), BF16)
    conv64 = O.conv(sd64, "conv_in", x.double())
    c = _plain_case(conv64 + kps_rows, (O.conv(sd16, "conv_in", x) + kps[idx]).double(), zero=kps_rows)
    y = ops.conv_in(x.cuda(), eng.W["conv_in.weight"], eng.W["conv_in.bias"], C0, addend=_tok(kps),
                    add_frame=idx.to(torch.int32).cuda() if frame_idx else None)
    torch.cuda.synchronize()
    assert not judge(f"conv_in + kps {'frame_idx' if frame_idx else 'in order'}", _img(y, B, H, H), c)


@pytest_gpu
@pytest.mark.parametrize("level", [0, 1, 2])
def test_downsample_conv(small, level):
    from vexpress_b200 import ops
    sd = small_sd()
    p = f"down_blocks.{level}.downsamplers.0.conv"
    eng = _load(small, _sub(sd, p + "."))
    C, H, B = CFG["block_out_channels"][level], 16 >> level, 8
    x = _frames(_gen("down", level), B, C, H, H)
    sd64, sd16 = _cast(_sub(sd, p + "."), F64), _cast(_sub(sd, p + "."), BF16)
    c = _plain_case(O.conv(sd64, p, x.double(), stride=2, padding=1), O.conv(sd16, p, x, stride=2, padding=1).double())
    y = ops.downsample_conv(_tok(x), B, H, H, eng.W[p + ".weight"], eng.W[p + ".bias"])
    torch.cuda.synchronize()
    assert not judge(f"downsample {p}", _img(y, B, H // 2, H // 2), c)


@pytest_gpu
@pytest.mark.parametrize("level", [0, 1, 2])
def test_upsample_conv(small, level):
    from vexpress_b200 import ops
    sd = small_sd()
    p = f"up_blocks.{level}.upsamplers.0.conv"
    eng = _load(small, _sub(sd, p + "."))
    C, H, B = list(reversed(CFG["block_out_channels"]))[level], 2 << level, 8
    x = _frames(_gen("up", level), B, C, H, H)
    sd64, sd16 = _cast(_sub(sd, p + "."), F64), _cast(_sub(sd, p + "."), BF16)
    up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")
    c = _plain_case(O.conv(sd64, p, up(x.double())), O.conv(sd16, p, up(x)).double())
    y = ops.upconv3x3(_tok(x).view(B, H, H, -1), eng.W[p + ".weight"], eng.W[p + ".bias"])
    torch.cuda.synchronize()
    assert not judge(f"upsample {p}", _img(y, B, 2 * H, 2 * H), c)


@pytest_gpu
@pytest.mark.parametrize("n", [1, 2])
def test_conv_norm_out_and_conv_out(small, n):
    from vexpress_b200 import ops
    sd = small_sd()
    sub = _sub(sd, "conv_norm_out.", "conv_out.")
    eng = _load(small, sub)
    B, H, C0 = 2 * n * 4, 16, CFG["block_out_channels"][0]
    x = _frames(_gen("out", n), B, C0, H, H)

    def run(sd_, xx):
        return O.conv(sd_, "conv_out", F.silu(O.group_norm(sd_, "conv_norm_out", xx, GROUPS, EPS)))
    c = _plain_case(run(_cast(sub, F64), x.double()), run(_cast(sub, BF16), x).double())
    h = eng._groupnorm(_tok(x), B, H * H, eng.W["conv_norm_out.weight"], eng.W["conv_norm_out.bias"], eng.eps, True, n=n)
    out = torch.empty((B, 4, H, H), device="cuda", dtype=BF16)
    ops.conv_out_tc(h, B, H, H, eng.W["conv_out.packed_w"], eng.W["conv_out.packed_b"], out)
    torch.cuda.synchronize()
    assert not judge(f"conv_norm_out + conv_out n={n}", out.double().cpu(), c)


# -------------------------------------------------------------------------------------------------------- ReferenceNet
@pytest.fixture(scope="module")
def refnet():
    from vexpress_b200.modules import UNet2DConditionModel
    sd = O.synth_state_dict(O.refnet_param_shapes(CFG), 4323)
    model = UNet2DConditionModel(block_out_channels=CFG["block_out_channels"],
                                 cross_attention_dim=CFG["cross_attention_dim"])
    model.load_state_dict(sd, strict=True)
    return sd, model.to(BF16).to("cuda")


@pytest_gpu
@pytest.mark.parametrize("branch", list(WRITE_BRANCHES))
def test_refnet_write_block(refnet, branch):
    """The bank the write pass stores (norm2 of h + attn1) and the block output, with one branch isolated."""
    sd, model = refnet
    p, H = "down_blocks.1.attentions.0", 8
    tb = p + ".transformer_blocks.0"
    sub = _sub(sd, p + ".")
    iso = isolate(sub, tb, WRITE_BRANCHES, branch, WRITE_GAIN.get(branch, 1.0))
    eng = _load(model, iso)
    C = sub[p + ".norm.weight"].shape[0]
    g = _gen("refnet", branch)
    x = _frames(g, 1, C, H, H)
    enc = _ln_rows(torch.randn(1, 1, CFG["cross_attention_dim"], generator=g))
    with torch.no_grad():
        ref, bank = O.transformer_2d_write(_cast(iso, F64), p, x.double(), enc.double(), HEADS, GROUPS)
        zero, _ = O.transformer_2d_write(_cast(isolate(sub, tb, WRITE_BRANCHES, branch, drop_keep=True), F64), p,
                                         x.double(), enc.double(), HEADS, GROUPS)
        eager, bank16 = O.transformer_2d_write(_cast(iso, BF16), p, x, enc, HEADS, GROUPS)
    c = _finish({}, ref, zero, eager.double(), x_res=x.double())
    assert c["share"] >= MIN_SHARE, (branch, c["share"])
    model.write_banks = True
    blk = model.get_submodule(tb)
    blk.bank = []
    y = eng._transformer_write(p, _tok(x), 1, H * H, enc.reshape(1, -1).cuda())
    torch.cuda.synchronize()
    assert len(blk.bank) == 1
    bad = [judge(f"refnet write {branch} output", _img(y, 1, H, H), c),
           judge(f"refnet write {branch} bank", blk.bank[0].double().cpu(), _plain_case(bank, bank16.double()))]
    assert not any(bad), "\n".join(b for b in bad if b)


# ---------------------------------------------------------------------------------------------------------------- VAE
VCFG = O.small_vae_cfg()


@pytest.fixture(scope="module")
def vae():
    from vexpress_b200.modules.vae import AutoencoderKL
    sd = O.synth_state_dict({**O.vae_param_shapes(VCFG), **O.vae_encoder_param_shapes(VCFG)}, 4324)
    model = AutoencoderKL(block_out_channels=VCFG["block_out_channels"], layers_per_block=VCFG["layers_per_block"])
    model.load_state_dict(sd, strict=True)
    return sd, model.to(BF16).to("cuda")


def _vae_engine(model, sd):
    with torch.no_grad():
        for k, v in sd.items():
            model.get_parameter(k).copy_(v)
    model._engine = model._enc_engine = None
    return model.engine()


@pytest_gpu
def test_vae_decoder_resnet(vae):
    sd, model = vae
    p = "decoder.up_blocks.2.resnets.0"                   # 128 -> 64 with conv_shortcut
    sub = _sub(sd, p + ".")
    eng = _vae_engine(model, sub)
    B, H = 2, 16
    x = _frames(_gen("vae-res"), B, 128, H, H)
    run = lambda s, xx: O._vae_resnet(s, p, xx, GROUPS)
    zero = run(_cast(isolate(sub, p, {"conv2": "conv2"}, "conv2", drop_keep=True), F64), x.double())
    c = _finish({}, run(_cast(sub, F64), x.double()), zero, run(_cast(sub, BF16), x).double())
    y = eng._res(p, _tok(x), B, H, H)
    torch.cuda.synchronize()
    assert not judge("vae decoder resnet (conv_shortcut)", _img(y, B, H, H), c)


@pytest_gpu
@pytest.mark.parametrize("side", ["decoder", "encoder"])
def test_vae_mid_attention(vae, side):
    sd, model = vae
    p = f"{side}.mid_block.attentions.0"
    sub = _sub(sd, p + ".")
    eng = _vae_engine(model, sub)
    if side == "encoder":
        from vexpress_b200.modules.vae import VaeEncoderEngine
        eng = VaeEncoderEngine(model)
    B, H, C = 2, 8, VCFG["block_out_channels"][-1]
    x = _frames(_gen("vae-attn", side), B, C, H, H)
    run = lambda s, xx: O._vae_attn(s, p, xx, GROUPS)
    c = _finish({}, run(_cast(sub, F64), x.double()), x.double(), run(_cast(sub, BF16), x).double())
    y = eng._attn(p, _tok(x), B, H * H)
    torch.cuda.synchronize()
    assert not judge(f"vae {side} mid attention", _img(y, B, H, H), c)


@pytest_gpu
def test_vae_upsampler(vae):
    from vexpress_b200 import ops
    sd, model = vae
    p = "decoder.up_blocks.1.upsamplers.0.conv"
    sub = _sub(sd, p + ".")
    eng = _vae_engine(model, sub)
    B, H, C = 2, 16, 128
    x = _frames(_gen("vae-up"), B, C, H, H)
    up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")
    c = _plain_case(O.conv(_cast(sub, F64), p, up(x.double())), O.conv(_cast(sub, BF16), p, up(x)).double())
    y = ops.upconv3x3(_tok(x).view(B, H, H, -1), eng.W[p + ".weight"], eng.W[p + ".bias"])
    torch.cuda.synchronize()
    assert not judge("vae upsampler", _img(y, B, 2 * H, 2 * H), c)


@pytest_gpu
def test_vae_encoder_downsampler(vae):
    """Downsample2D(padding=0): pad (0, 1, 0, 1), then the stride-2 conv."""
    from vexpress_b200 import ops
    from vexpress_b200.modules.vae import VaeEncoderEngine
    sd, model = vae
    p = "encoder.down_blocks.1.downsamplers.0.conv"
    sub = _sub(sd, p + ".")
    _vae_engine(model, sub)
    eng = VaeEncoderEngine(model)
    B, H, C = 2, 16, VCFG["block_out_channels"][1]
    x = _frames(_gen("vae-down"), B, C, H, H)
    run = lambda s, xx: O.conv(s, p, F.pad(xx, (0, 1, 0, 1)), stride=2, padding=0)
    c = _plain_case(run(_cast(sub, F64), x.double()), run(_cast(sub, BF16), x).double())
    y = ops.downsample_conv(_tok(x), B, H, H, eng.W[p + ".weight"], eng.W[p + ".bias"], pad_lo=0)
    torch.cuda.synchronize()
    assert not judge("vae encoder downsampler", _img(y, B, H // 2, H // 2), c)


@pytest_gpu
@pytest.mark.parametrize("post", [False, True])
def test_vae_decode_pre_scale_post(vae, post):
    """decode() with the 1 / 0.18215 pre-scale fused into conv_in, with and without the (x / 2 + 0.5).clamp(0, 1) post."""
    sd, model = vae
    sub = _sub(sd, "decoder.", "post_quant_conv.")
    eng = _vae_engine(model, sub)
    z = (0.18215 * torch.randn(2, 4, 8, 8, generator=_gen("vae-decode", post))).to(BF16)

    def run(s, zz):
        img = O.vae_decode(s, VCFG, zz * (1 / 0.18215))
        return (img / 2 + 0.5).clamp(0, 1) if post else img
    with torch.no_grad():
        c = _plain_case(run(_cast(sub, F64), z.double()), run(_cast(sub, BF16), z).double())
    out = eng.decode(z.cuda(), pre_scale=1 / 0.18215, post=post, out_dtype=torch.float32)
    torch.cuda.synchronize()
    assert not judge(f"vae decode post={post}", out.double().cpu(), c)
