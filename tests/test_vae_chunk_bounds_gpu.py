"""The VAE decoder at the batch the pipeline decodes: 16 frames per launch (``VExpressPipeline.vae_chunk``) at 512 x 512
and 768 x 768 (64 x 64 and 96 x 96 latents), every kernel against an fp64 reference, frame by frame.

Two things change between the one- and two-frame cases of the sibling files and the 16-frame chunk.  GroupNorm's chunking
does: ``ops._gn_S`` gives each frame min(HW / 32, capacity / NB, 64) pixel chunks, so at NB = 16 every thread's fp32 add
chain is several times longer than at NB = 1, and the one-launch / two-kernel choice is re-made for that grid.  And offsets
pass 2^31: at 768 x 768 the upsampler of up block 2 writes 16 x 768^2 x 256 bf16 elements (more than 2^31), and the
128-channel 768^2 and 512-channel 384^2 tensors pass 2^31 bytes.

1. Case list (CPU).  ``_RecordingOps`` (tests/test_host_cpu._ShapeOps plus softmax_rows) stands in for ``ops`` while
   ``VaeDecoderEngine.decode`` runs the full-width decoder (oracle VAE_CFG: 512 / 512 / 256 / 128 channels) on the meta
   device, in the pipeline's ``decode_latents`` form: 16 latent frames, pre_scale 1 / 0.18215, post = True, fp32 output into
   frames 16..31 of a (3, 48, H, W) video view.  Every call is normalised to a key that includes NB (``_call_key``); every
   recorded key must have a GPU case here and every case-table entry must cover a recorded key
   (``test_decoder_calls_at_chunk_16_are_covered``).  The recording also lists, per size, the frames that hold element 2^31
   or byte 2^31 of an operand or output: {0, 7, 14, 15} at 768 x 768, none at 512 x 512 (its largest tensor, 256 channels
   at 512^2, is exactly 2^31 bytes).

2. Kernel cases (GPU), judged by the sibling files' references and bounds, unchanged: ``groupnorm_ref64`` / ``_gn_adds``
   (tests/test_norm_bounds_gpu.py) and ``conv_cols`` / ``linear_ref64`` / ``linear_bound`` / ``bound_check`` /
   ``_conv_in_ref64`` (tests/test_gemm_bounds_gpu.py), applied one frame (and one row or channel-group chunk of it) at a
   time, so that the fp64 temporaries stay a few GB where a whole-batch reference would need tens.  Inputs are drawn frame by
   frame in bf16 from per-frame seeds; GroupNorm frames also get their own scale 2^(n mod 4 - 1) and offset (n - 7.5) / 2,
   so statistics of one frame applied to another leave the bound.  Inputs are interior views of NaN-bordered buffers (the
   convolutions' inputs: frames 1..16 of a buffer whose frames 0 and 17 are NaN), outputs go inside sentinel borders that
   must survive.
   * GroupNorm through the default dispatch, with the bound's add count taken at the S the dispatch used
     (``_gn_path``); the same input through that path's own entry point must give the same bits (which proves the path
     and S).  The tail chunk of a video has 1..15 frames: every distinct (S, path) those produce runs as well.
   * conv3x3 (+ the 1x1 shortcut as residual), upconv3x3 (per frame and parity class), the shortcut / q / k / to_out
     GEMMs at M = 16 HW, the per-frame scores / V^T / P V GEMMs and softmax_rows on frame 15's row slice, conv_in with
     pre_scale and post_quant_conv, conv_out_tc with post into frames 16..31 of a sentinel-filled fp32 (3, 48, H, W) video.

3. The composed decoder (GPU): 16 distinct latent frames through ``AutoencoderKL.decode_latents`` at both sizes; frames
   0, 15 and every frame the recording lists in 1. are compared with the oracle decoding that frame alone, in fp64 (the
   reference) and bf16 (the yardstick), by tests/test_size768_bounds_gpu's criterion e_prod <= 1.5 e_eager + 2e-3.

4. Self-test (CPU): ``test_frame_judges_reject_cross_frame_faults`` runs torch models through the same per-frame judges:
   a conv whose frame n reads frame n - 1, GroupNorm with the statistics of frame n - 1, and GroupNorm statistics whose
   add chain is one S-step longer than the bound accounts for (``_gn_worst_case``) must be rejected; the faithful models
   must pass.

No case holds more than 40 GiB of device memory at once (``_case_peak``): the GPU is shared.
"""
import functools
import math
import time

import pytest
import torch

from test_gemm_bounds_gpu import (_INNER, _SENTINEL32, _block_exp, _border_untouched, _bordered, _conv_in_ref64, _seed,
                                  _sentinel_buf, bound_check, conv_cols, conv_inputs, emulate_gemm, gemm_inputs,
                                  linear_bound, linear_ref64)
from test_host_cpu import _ShapeOps
from test_norm_bounds_gpu import (GN_FAMILIES, _cluster_fits, _gn_adds, emulate_groupnorm, gn_inputs, groupnorm_ref64,
                                  softmax_ref64)

CHUNK = 16                   # VExpressPipeline.vae_chunk: frames per decoder launch
LATENTS = (64, 96)           # latent sides of 512 x 512 and 768 x 768 videos
EPS = 1e-6
SCALING = 0.18215
_BUDGET = 1 << 31            # bytes of fp64 temporaries per reference chunk


# ---------------------------------------------------------------------------------------------------------- case tables
def _gn_table(h):
    """(NB, HW, C, silu): mid block and up block 0 (512 ch at h^2; without SiLU: the attention's group_norm), up block 1
    (512 at 4 h^2), up block 2 (512 -> 256 at 16 h^2), up block 3 (256 -> 128 at 64 h^2) and conv_norm_out."""
    return [(CHUNK, (m * h) ** 2, c, silu) for m, c, silu in
            ((1, 512, True), (1, 512, False), (2, 512, True), (4, 512, True), (4, 256, True), (8, 256, True),
             (8, 128, True))]


GROUPNORM = [e for h in LATENTS for e in _gn_table(h)]
# (NB, H, W, C, Cout, residual): conv1 (no residual) and conv2 (+ the block input or its 1x1 shortcut) of every resnet
CONV3X3 = [(CHUNK, m * h, m * h, c, co, res) for h in LATENTS for m, c, co, res in
           ((1, 512, 512, False), (1, 512, 512, True), (2, 512, 512, False), (2, 512, 512, True), (4, 512, 256, False),
            (4, 256, 256, False), (4, 256, 256, True), (8, 256, 128, False), (8, 128, 128, False), (8, 128, 128, True))]
# (NB, H, W, C, Cout) of the three upsamplers (input size)
UPCONV = [(CHUNK, m * h, m * h, c, c) for h in LATENTS for m, c in ((1, 512), (2, 512), (4, 256))]
# (M, K, N, residual, kind) of the GEMMs over all 16 frames: the two 1x1 shortcuts, the mid-block attention's q / k
# (one key) and to_out (+ residual)
GEMM_ROWS = [(CHUNK * hw, k, n, res, kind) for h in LATENTS
             for hw, k, n, res, kind in ((16 * h * h, 512, 256, False, "shortcut"), (64 * h * h, 256, 128, False, "shortcut"),
                                         (h * h, 512, 512, False, "q/k"), (h * h, 512, 512, True, "to_out"))]
# HW of the mid-block attention: per frame, scores (fp32 out), softmax_rows, V^T = Wv xn^T and P V
ATTENTION = [h * h for h in LATENTS]
CONV_IN = [(CHUNK, h, h, 512) for h in LATENTS]                     # post_quant_conv + pre_scale, 4 -> 512
CONV_OUT = [(CHUNK, 8 * h, 8 * h, 128, 3) for h in LATENTS]         # 128 -> 3, post, fp32 video view
C_ATT = 512


def _case_keys():
    """{call key (``_call_key``) -> the table entry that covers it}; an ATTENTION entry stands for its three GEMMs and
    softmax_rows, a q/k GEMM_ROWS entry for both projections."""
    keys = {}

    def add(key, entry):
        assert key not in keys, (key, entry, keys[key])
        keys[key] = entry
    for NB, hw, c, silu in GROUPNORM:
        add(("groupnorm", NB, hw, c, 0, EPS, silu), ("GROUPNORM", NB, hw, c, silu))
    for NB, H, W, c, co, res in CONV3X3:
        add(("conv3x3", NB, H, W, c, co, res), ("CONV3X3", NB, H, W, c, co, res))
    for NB, H, W, c, co in UPCONV:
        add(("upconv3x3", NB, H, W, c, co), ("UPCONV", NB, H, W, c, co))
    for M, K, N, res, kind in GEMM_ROWS:
        add(("gemm", M, K, N, res, False, False), ("GEMM_ROWS", M, K, N, res, kind))
    for hw in ATTENTION:
        e = ("ATTENTION", hw)
        add(("gemm", hw, C_ATT, hw, False, True, True), e)           # scores = q k^T (k: activations as W)
        add(("gemm", C_ATT, C_ATT, hw, False, False, True), e)       # V^T = Wv xn^T (xn: activations as W)
        add(("gemm", hw, hw, C_ATT, False, False, True), e)          # P V (V^T: activations as W)
        add(("softmax_rows", hw), e)
    for NB, H, W, co in CONV_IN:
        add(("conv_in", NB, H, W, co, True), ("CONV_IN", NB, H, W, co))
    for NB, H, W, c, co in CONV_OUT:
        add(("conv_out_tc", NB, H, W, c, co, True, "float32"), ("CONV_OUT", NB, H, W, c, co))
    return keys


def _call_key(op, a, k, weights):
    """The normal form of one ops call of ``VaeDecoderEngine.decode``; ``weights``: ids of the engine's packed tensors."""
    if op == "groupnorm":
        x1, NB, HW, x2 = a[0], a[1], a[2], k.get("x2")
        return ("groupnorm", NB, HW, x1.shape[1], 0 if x2 is None else x2.shape[1], a[5], bool(a[6]))
    if op == "conv3x3":
        NB, H, W, C = a[0].shape
        assert k.get("bias2") is None and k.get("scale", 1.0) == 1.0
        return ("conv3x3", NB, H, W, C, a[1].shape[0], k.get("residual") is not None)
    if op == "upconv3x3":
        NB, H, W, C = a[0].shape
        return ("upconv3x3", NB, H, W, C, a[1].shape[0] // 4)
    if op == "gemm":
        x, w = a[0], a[1]
        assert k.get("a2") is None and k.get("bias2") is None and not k.get("geglu")
        return ("gemm", x.shape[0], x.shape[1], w.shape[0], k.get("residual") is not None, bool(k.get("out_f32")),
                id(w) not in weights)
    if op == "softmax_rows":
        return ("softmax_rows", a[0].shape[1])
    if op == "conv_in":
        NB, _, H, W = a[0].shape
        assert k.get("pre_w") is None or k.get("pre_scale") == 1 / SCALING
        return ("conv_in", NB, H, W, a[3], k.get("pre_w") is not None)
    if op == "conv_out_tc":
        x, NB, H, W, out = a[0], a[1], a[2], a[3], a[6]
        return ("conv_out_tc", NB, H, W, x.shape[1], out.shape[1], bool(k.get("post")), str(out.dtype).split(".")[-1])
    raise AssertionError(f"ops.{op}: the decoder makes a call this file has no family for")


class _RecordingOps(_ShapeOps):
    """_ShapeOps (with softmax_rows) that records the key of every call, and the frames holding element or byte 2^31 of
    any operand or output past that size (those tensors are [NB ..., ...] frame-major)."""

    def __init__(self, weights):
        super().__init__()
        self.weights = weights
        self.seen = {}
        self.big = {}               # latent side -> {frame: [what]}
        self.h = None

    def _note(self, op, t, NB):
        for off, unit in ((1 << 31, "element"), ((1 << 31) // t.element_size(), "byte")):
            if off < t.numel():
                assert t.shape[0] % NB == 0, (op, tuple(t.shape))
                n = off // (t.numel() // NB)
                self.big.setdefault(self.h, {}).setdefault(n, []).append(f"{unit} 2^31 of ops.{op} {tuple(t.shape)}")

    def __getattr__(self, op):
        run = super().__getattr__(op) if op != "softmax_rows" else (
            lambda x, out=None: out if out is not None else torch.zeros(x.shape, dtype=torch.bfloat16))

        def rec(*a, **k):
            key = _call_key(op, a, k, self.weights)
            self.seen.setdefault(key, (op, [tuple(t.shape) for t in a if torch.is_tensor(t)]))
            res = run(*a, **k)
            if torch.is_tensor(res) and res.dtype == torch.float32 and not k.get("out_f32") and op != "conv_out_tc":
                res = res.bfloat16()        # what the real wrapper returns (_ShapeOps allocates fp32)
            outs = list(res) if isinstance(res, tuple) else [res]
            for t in list(a) + list(k.values()) + outs:
                if torch.is_tensor(t) and t.numel() * t.element_size() > (1 << 31):
                    self._note(op, t, CHUNK)
            return res
        return rec


def _meta_engine():
    """The full-width VaeDecoderEngine with its weights packed on the meta device (shapes only; no kernel runs)."""
    from oracle import vx_oracle as O
    from vexpress_b200.modules import vae as V
    cfg = O.VAE_CFG
    with torch.device("meta"):
        model = V.AutoencoderKL(block_out_channels=cfg["block_out_channels"], layers_per_block=cfg["layers_per_block"],
                                with_encoder=False).to(torch.bfloat16)
        eng = object.__new__(V.VaeDecoderEngine)
        eng.model, eng.dev = model, torch.device("meta")
        eng.boc, eng.layers = tuple(model.config["block_out_channels"]), model.config["layers_per_block"]
        eng.W = {}
        eng._pack(model.state_dict())
    return eng


@functools.lru_cache(maxsize=None)
def _recorded():
    """(seen, big) of the decode_latents form at every size in LATENTS (module docstring, section 1)."""
    from vexpress_b200.modules import vae as V
    eng = _meta_engine()
    fake = _RecordingOps({id(t) for t in eng.W.values()})
    with pytest.MonkeyPatch.context() as mp, torch.device("meta"):
        mp.setattr(V, "ops", fake)
        for h in LATENTS:
            fake.h = h
            z = torch.empty(CHUNK, 4, h, h, dtype=torch.bfloat16)
            video = torch.empty(3, 3 * CHUNK, 8 * h, 8 * h)
            out = eng.decode(z, pre_scale=1 / SCALING, post=True, out_dtype=torch.float32,
                             out=video[:, CHUNK:2 * CHUNK].permute(1, 0, 2, 3))
            assert out.shape == (CHUNK, 3, 8 * h, 8 * h)
    return fake.seen, fake.big


def _big_frames(h):
    return {n: v for n, v in _recorded()[1].get(h, {}).items()}


def test_decoder_calls_at_chunk_16_are_covered():
    """Every ops call of the 16-frame decoder at 64 x 64 and 96 x 96 latents has a GPU case here, and every case-table
    entry covers a call the decoder makes (so removing any entry fails, naming the key it covered)."""
    seen, big = _recorded()
    cases = _case_keys()
    for k in sorted(seen, key=str):
        print(("   " if k in cases else "!! ") + str(k))
    missing = {k: v for k, v in seen.items() if k not in cases}
    assert not missing, "decoder calls without a GPU case:\n" + "\n".join(f"{k}: {v}" for k, v in missing.items())
    stale = {k: e for k, e in cases.items() if k not in seen}
    unused = {e for e in stale.values()} - {cases[k] for k in seen}
    assert not unused, "case-table entries no decoder call needs:\n" + "\n".join(
        f"{e}: covers {[k for k, v in stale.items() if v == e]}" for e in sorted(unused, key=str))
    for h in LATENTS:
        for n, what in sorted(big.get(h, {}).items()):
            print(f"{8 * h} x {8 * h}: frame {n} holds " + "; ".join(sorted(set(what))))
    assert sorted(_big_frames(96)) == [7, 14] and not _big_frames(64), {h: sorted(_big_frames(h)) for h in LATENTS}
    print(f"{len(seen)} call forms recorded, all covered by {len(set(cases.values()))} table entries")


# ------------------------------------------------------------------------------------------------- per-frame judging
class _Frames:
    """Worst bound ratio (with its frame and place) and the global relative error of one case, accumulated over frames
    and chunks of frames."""

    def __init__(self, family, case, fam):
        self.family, self.case, self.fam = family, case, fam
        self.worst, self.where, self.err2, self.ref2, self.net2 = 0.0, "", 0.0, 0.0, 0.0
        self.bad = []

    def add(self, frame, out, ref, bnd, bf16_out=True, residual=None, what=""):
        worst, _, where = bound_check(out, ref, bnd, bf16_out)
        o = out.double().reshape(ref.shape)
        self.err2 += float((o - ref).norm()) ** 2
        self.ref2 += float(ref.norm()) ** 2
        if residual is not None:
            self.net2 += float((ref - residual.double()).norm()) ** 2
        if worst > self.worst or not self.where:
            self.worst, self.where = worst, f"frame {frame}{what}: {where}"
        if torch.isnan(o).any():
            self.bad.append(f"frame {frame}{what}: NaN in the output")

    def finish(self, border=""):
        """Prints the case, records the family's worst ratio -> '' or the failure message."""
        scale = math.sqrt(max(self.ref2, self.net2))
        rel = math.sqrt(self.err2) / scale if scale > 0 else math.sqrt(self.err2)
        print(f"{self.family:18s} {self.case} {self.fam:9s}: worst ratio {self.worst:.3f} ({self.where[:40]}...), "
              f"rel {rel:.2e}")
        if self.worst > _WORST.get(self.family, (-1.0, ""))[0]:
            _WORST[self.family] = (self.worst, f"{self.case} {self.fam}, {self.where}")
        _REL[self.family] = max(_REL.get(self.family, 0.0), rel)
        bad = list(self.bad)
        if not self.worst <= 1:
            bad.append(f"bound exceeded, {self.where}")
        if not rel < 5e-3:
            bad.append(f"global rel {rel:.3e}")
        if border:
            bad.append(border)
        return f"{self.family} {self.case} {self.fam}: " + "; ".join(bad) if bad else ""


def _rows(rows, K, N):
    step = max(1, _BUDGET // (8 * (K + 6 * N)))
    return [(r0, min(rows, r0 + step)) for r0 in range(0, rows, step)]


def _judge_linear(j, frame, cols, out, w, bias=None, residual=None, scale=1.0, what=""):
    """One frame (or parity class) of a GEMM-shaped op: rows of ``cols`` [rows, K] (the exact operand values) against
    ``out`` [rows, N], row chunk by row chunk."""
    K, N = cols.shape[1], w.shape[0]
    for r0, r1 in _rows(cols.shape[0], K, N):
        res = None if residual is None else residual[r0:r1]
        ref, ref_abs, prod = linear_ref64(cols[r0:r1], w, bias, scale=scale, residual=res)
        j.add(frame, out[r0:r1], ref, linear_bound(ref, ref_abs, prod, K), residual=res, what=what)


def _judge_conv_frames(j, x, w, b, out, residual=None):
    """conv3x3 of NHWC x [NB, H, W, C] against out [NB H W, Cout], each frame against a reference of that frame alone."""
    NB, H, W, C = x.shape
    hw = H * W
    for n in range(NB):
        cols = conv_cols(x[n:n + 1]).reshape(hw, 9 * C)
        _judge_linear(j, n, cols, out[n * hw:(n + 1) * hw], w, b,
                      None if residual is None else residual[n * hw:(n + 1) * hw])


def _gn_chunks(HW, C, G=32):
    """Channel-group slices of a frame whose fp64 reference temporaries stay within the budget (groups are independent)."""
    cpg = C // G
    gs = max(1, min(G, _BUDGET // (12 * 8 * HW * cpg)))
    return [(g0 * cpg, min(G, g0 + gs) * cpg, min(G, g0 + gs) - g0) for g0 in range(0, G, gs)]


def _judge_gn_frames(j, x, NB, HW, gam, bet, eps, silu, n_add, out, bf16_out=True, G=32):
    """Per-frame GroupNorm of x [NB HW, C] against out, each frame (and group slice) against its own fp64 reference with
    the bound at ``n_add`` fp32 adds."""
    C = x.shape[1]
    for n in range(NB):
        r = slice(n * HW, (n + 1) * HW)
        for c0, c1, g in _gn_chunks(HW, C, G):
            ref, bnd = groupnorm_ref64(x[r, c0:c1], None, 1, HW, g, gam[c0:c1], bet[c0:c1], eps, silu, n_add)
            j.add(n, out[r, c0:c1], ref, bnd, bf16_out, what=f" channels {c0}..{c1}")


def _gn_frame_affine(x, n):
    """Frame n's own scale 2^(n mod 4 - 1) and offset (n - 7.5) / 2, rounded to bf16."""
    return (x.float() * 2.0 ** (n % 4 - 1) + 0.5 * (n - 7.5)).bfloat16()


# ------------------------------------------------------------------------------------------- CPU self-test (section 4)
def _gn_worst_case(x, NB, HW, gam, bet, eps, chain, G=32):
    """GroupNorm in fp64 whose per-group sums of x - pivot carry the largest error a chain of ``chain`` fp32 adds may give
    (``chain`` u sum |addend|, for both the sum and the sum of squares), in the direction that moves M2 most; no output
    rounding.  With the pivot at the group's farthest value and every x - pivot of one sign, that is the error the bound's
    n_add term allows for, so the bound at n_add = chain passes it and a bound at a smaller n_add must not."""
    xd = x.double().view(NB, HW, G, -1)
    piv = xd[:, :1, :, :1]
    d = xd - piv
    N = HW * d.shape[-1]
    A, Q = d.sum((1, 3)), (d * d).sum((1, 3))
    e = chain * 2.0 ** -24
    A = A - torch.sign(A) * e * d.abs().sum((1, 3))
    Q = Q + e * Q
    mean = A / N + piv.view(NB, G)
    rstd = ((Q - A * A / N) / N + eps).rsqrt()
    y = (xd - mean[:, None, :, None]) * rstd[:, None, :, None]
    return (y.reshape(NB * HW, -1) * gam.double() + bet.double())


def _two_point_frames(NB, HW, C, k2, g):
    """Every group: a fraction 1 / (1 + k2) of zeros (pixel 0 of its first channel among them), ones elsewhere, times a
    per-frame scale: max (x - mu)^2 / var = k2, the pivot is the farthest value and every x - pivot >= 0."""
    x = (torch.rand(NB, HW, C, generator=g) >= 1 / (1 + k2)).float()
    x[:, 0] = 0.0
    return (x * 2.0 ** (torch.arange(NB) % 4 - 1.0)[:, None, None]).reshape(NB * HW, C).bfloat16()


def test_frame_judges_reject_cross_frame_faults():
    """The per-frame judges the GPU cases use reject a conv whose frame n reads frame n - 1's input, GroupNorm with the
    statistics of frame n - 1, and statistics accumulated over a chunk one S-step longer than the bound's S (worst-case
    rounding: an n_add that is too small must not pass silently); the faithful models pass."""
    g = torch.Generator().manual_seed(31)
    NB = CHUNK
    # conv: frame n from frame n - 1's input
    H, W, C, Co = 4, 6, 64, 32
    x = torch.randn(NB, H, W, C, generator=g).bfloat16()
    _, w, b, _ = conv_inputs("flat", g, 1, 1, 1, C, Co)
    res = torch.randn(NB * H * W, Co, generator=g).bfloat16()
    verdict = {}
    for name, xin in (("faithful", x), ("frame n reads frame n - 1", x.roll(1, 0))):
        out = emulate_gemm(conv_cols(xin).reshape(-1, 9 * C), w, b, residual=res)
        j = _Frames("conv3x3", f"NB {NB} {H}x{W} C {C}->{Co}", name[:9])
        _judge_conv_frames(j, x, w, b, out, res)
        verdict[f"conv {name}"] = j.finish()
    # GroupNorm with per-frame scale and offset, at an S the dispatch picks at NB = 16 (capacity / 16 on a device that
    # keeps 64 GroupNorm CTAs resident: S = 4)
    HW, C, S = 256, 64, 4
    frames = [_gn_frame_affine(gn_inputs("flat", g, 1, HW, C, 0)[0], n) for n in range(NB)]
    x = torch.cat(frames)
    _, _, gam, bet = gn_inputs("flat", g, 1, 32, C, 0)
    n_add = _gn_adds(HW, C, 32, S)
    rev = lambda t: t.view(NB, HW, C).flip(0).reshape(NB * HW, C)
    for name, out in (("faithful", emulate_groupnorm(x, None, NB, HW, 32, gam, bet, EPS, True, S)),
                      # the model's frame_shift gives frame n the statistics of frame n + 1; on the reversed batch that
                      # is frame n - 1 of the original order
                      ("stats of frame n - 1", rev(emulate_groupnorm(rev(x), None, NB, HW, 32, gam, bet, EPS, True, S,
                                                                     "frame_shift")))):
        j = _Frames("groupnorm", f"NB {NB} HW {HW} C {C} S {S}", name[:9])
        _judge_gn_frames(j, x, NB, HW, gam, bet, EPS, True, n_add, out)
        verdict[f"groupnorm {name}"] = j.finish()
    # worst-case rounding of the statistics: 32768 pixels of 64 channels in S = 8 chunks (the chunk term dominates the add
    # count), k2 = 100 (the relative variance error stays ~0.5 %: the bound's first-order form holds)
    HW, S = 32768, 8
    x = _two_point_frames(2, HW, C, 100.0, g)
    gam, bet = 1 + 0.1 * torch.rand(C, generator=g), 0.1 * torch.rand(C, generator=g)
    n_add = _gn_adds(HW, C, 32, S)
    for name, chain in (("faithful", n_add), ("chunk one S-step longer", _gn_adds(HW, C, 32, S - 1))):
        j = _Frames("groupnorm", f"NB 2 HW {HW} C {C} S {S}", name[:9])
        _judge_gn_frames(j, x, 2, HW, gam, bet, EPS, False, n_add, _gn_worst_case(x, 2, HW, gam, bet, EPS, chain),
                         bf16_out=False)
        verdict[f"groupnorm worst case, {name} (n_add {chain} against {n_add})"] = j.finish()
    for k, v in verdict.items():
        print(f"{k}: {v or 'passes'}")
    for k, v in verdict.items():
        assert bool(v) == ("faithful" not in k), (k, v)


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


_WORST = {}                  # op family -> (worst bound ratio, case and place)
_REL = {}                    # op family -> largest global relative error
_GN = []                     # GroupNorm (S, path) lines
_NET = []                    # composed-decoder lines
_PEAK = {}                   # case -> peak device memory (GiB)
PEAK_GIB = 40.0              # the file shares its GPU: no case may hold more than this at once


@pytest.fixture(scope="module", autouse=True)
def _summary():
    """Prints, at the end of the module: the worst bound ratio and largest global relative error per family, the GroupNorm
    paths, the composed-decoder ratios, the peak memory per case and the file's wall time."""
    t0 = time.time()
    yield
    for fam, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {fam:18s} {worst:.3f}, global rel {_REL[fam]:.2e}  ({case})")
    for row in _GN + _NET:
        print(row)
    for name, peak in sorted(_PEAK.items(), key=lambda kv: -kv[1]):
        print(f"peak device memory {peak:6.2f} GiB  {name}")
    if _PEAK:
        print(f"vae chunk file: {time.time() - t0:.1f} s")


@pytest.fixture(autouse=True)
def _case_peak(request):
    """Peak device memory of each GPU case, printed at the end of the file and held under PEAK_GIB."""
    if request.node.get_closest_marker("gpu") is None or not torch.cuda.is_available():
        yield
        return
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    _PEAK[request.node.name] = peak
    assert peak <= PEAK_GIB, f"{request.node.name}: peak device memory {peak:.2f} GiB"


def _gen(*ints):
    return torch.Generator(device="cuda").manual_seed(_seed(*ints))


FAMS = ("flat", "blocks", "frames")
_FI = {"flat": 0, "blocks": 1, "frames": 3}      # test_gemm_bounds_gpu.FAMILIES indices


def _act_frame(fam, seed, n, rows, K):
    """Frame n's activations [rows, K] (bf16): N(0, 1) from the frame's own seed; blocks: 64-wide K blocks scaled 2^+-6
    (the weights of the case inversely); frames: scaled 4^(n mod 3)."""
    a = torch.randn(rows, K, device="cuda", generator=_gen(seed, n))
    if fam == "blocks":
        a *= torch.exp2(_block_exp(K)).cuda()
    if fam == "frames":
        a *= 4.0 ** (n % 3)
    return a.bfloat16()


# ---- GroupNorm
def _gn_path(ops, NB, HW, C):
    """(S, path) of ops.groupnorm: the cluster kernel (S 1) where the frame fits a cluster, else the one-launch kernel,
    whose NB * S CTAs fit the capacity _gn_S sizes S by (the smaller of its and the apply kernel's occupancy), else the
    statistics / apply pair."""
    if ops._GN_CLUSTER and _cluster_fits(NB, HW, C):
        return 1, "cluster"
    S = ops._gn_S(NB, HW, C)
    return S, "fused" if ops._GN_FUSED and NB * S <= ops._GN_CAP[C] else "pair"


def _run_gn(ops, fams, NB, HW, C, silu):
    """ops.groupnorm of each family over NB frames; the first family also through the chosen path's own entry point,
    which must give the same bits."""
    from test_norm_bounds_gpu import _gn_run
    S, path = _gn_path(ops, NB, HW, C)
    n_add = _gn_adds(HW, C, 32, S)
    case = f"NB {NB} HW {HW} C {C} silu {int(silu)} {path} S {S}"
    fails = []
    for i, fam in enumerate(fams):
        seed = _seed(NB, HW, C, silu, GN_FAMILIES.index(fam))
        xbuf, x = _bordered(NB * HW, C)
        for n in range(NB):
            x[n * HW:(n + 1) * HW] = _gn_frame_affine(gn_inputs(fam, _gen(seed, n), 1, HW, C, 0)[0], n)
        _, _, gam, bet = gn_inputs(fam, _gen(seed, NB), 1, 32, C, 0)
        obuf, out = _bordered(NB * HW, C)
        ops.groupnorm(x, NB, HW, gam, bet, EPS, silu, out=out)
        if i == 0:
            tbuf, twin = _bordered(NB * HW, C)
            rc, S2, ws = _gn_run(ops, path, x, None, NB, HW, gam, bet, EPS, silu, twin)
            torch.cuda.synchronize()
            assert rc == 0 and S2 == S and torch.equal(out.view(torch.int16), twin.view(torch.int16)), \
                f"{case}: the dispatch did not compute what {path} at S {S} computes (rc {rc}, S {S2})"
            del tbuf, twin, ws
        torch.cuda.synchronize()
        j = _Frames("groupnorm", case, fam)
        _judge_gn_frames(j, x, NB, HW, gam, bet, EPS, silu, n_add, out)
        fails.append(j.finish(_border_untouched(obuf, _INNER)))
        del xbuf, x, obuf, out
    return [f for f in fails if f]


def _gn_fams(silu):
    return ("flat", "offset", "silu-tail") if silu else ("flat", "offset")


@pytest.mark.gpu
@pytest.mark.parametrize("NB,HW,C,silu", GROUPNORM)
def test_groupnorm_chunk_within_bound(ops, NB, HW, C, silu):
    S, path = _gn_path(ops, NB, HW, C)
    _GN.append(f"groupnorm NB {NB} HW {HW} C {C}: {path}, S {S}, n_add {_gn_adds(HW, C, 32, S)} "
               f"(NB 1: S {_gn_path(ops, 1, HW, C)[0]}, n_add {_gn_adds(HW, C, 32, _gn_path(ops, 1, HW, C)[0])})")
    fails = _run_gn(ops, _gn_fams(silu), NB, HW, C, silu)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("h", LATENTS)
def test_groupnorm_tail_chunks_within_bound(ops, h):
    """The last chunk of a video holds 1..15 frames: every (S, path) such a chunk gets at a VAE (HW, C), other than the
    16-frame one, runs once (at the fewest frames that produce it)."""
    fails = []
    for HW, C in sorted({(hw, c) for _, hw, c, _ in _gn_table(h)}):
        tails = {}
        for NB in range(1, CHUNK + 1):
            tails.setdefault(_gn_path(ops, NB, HW, C), NB)
        tails.pop(_gn_path(ops, CHUNK, HW, C), None)
        _GN.append(f"groupnorm tail chunks HW {HW} C {C}: " + ", ".join(f"NB {nb}: {p} S {s}"
                                                                       for (s, p), nb in sorted(tails.items(),
                                                                                                key=lambda kv: kv[1])))
        for (S, path), NB in sorted(tails.items(), key=lambda kv: kv[1]):
            fails += _run_gn(ops, _gn_fams(True), NB, HW, C, True)
    assert not fails, "\n".join(fails)


# ---- 3x3 convolution and the folded upsample
def _conv_weights(fam, seed, C, Cout, taps):
    _, w, b, _ = conv_inputs(fam, _gen(seed, -1), 1, 1, 1, C, Cout, taps)
    return w, b


def _nan_frames(fam, seed, NB, H, W, C):
    """Frames 1..NB of a buffer whose frames 0 and NB + 1 are NaN, drawn frame by frame -> (buffer, view)."""
    xb = _sentinel_buf((NB + 2, H, W, C))
    for n in range(NB):
        xb[n + 1] = _act_frame(fam, seed, n, H * W, C).view(H, W, C)
    return xb, xb[1:NB + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout,res", CONV3X3)
def test_conv3x3_chunk_within_bound(ops, NB, H, W, C, Cout, res):
    """conv3x3 with bias, and (res) with the residual the resnet adds: the block input or its 1x1 shortcut."""
    hw = H * W
    fails = []
    for fam in FAMS:
        seed = _seed(NB, H, W, C, Cout, res, _FI[fam])
        w, b = _conv_weights(fam, seed, C, Cout, 9)
        xb, x = _nan_frames(fam, seed, NB, H, W, C)
        rbuf, r = _bordered(NB * hw, Cout) if res else (None, None)
        for n in range(NB if res else 0):
            r[n * hw:(n + 1) * hw] = torch.randn(hw, Cout, device="cuda", generator=_gen(seed, NB + n)).bfloat16()
        obuf, out = _bordered(NB * hw, Cout)
        ops.conv3x3(x, w, b, residual=r, out=out)
        torch.cuda.synchronize()
        j = _Frames("conv3x3" + (" + residual" if res else ""), f"NB {NB} {H}x{W} C {C}->{Cout}", fam)
        _judge_conv_frames(j, x, w, b, out, r)
        fails.append(j.finish(_border_untouched(obuf, _INNER)))
        del xb, x, rbuf, r, obuf, out
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,Cout", UPCONV)
def test_upconv3x3_chunk_within_bound(ops, NB, H, W, C, Cout):
    """conv3x3(upsample2x(x)): every frame's four parity classes against their 2x2 convolutions."""
    fails = []
    for fam in FAMS:
        seed = _seed(NB, H, W, C, Cout, 4, _FI[fam])
        w4, b = _conv_weights(fam, seed, C, 4 * Cout, 4)
        b = b[:Cout].contiguous()
        xb, x = _nan_frames(fam, seed, NB, H, W, C)
        obuf, out = _bordered(NB * 4 * H * W, Cout)
        ops.upconv3x3(x, w4, b, out=out)
        torch.cuda.synchronize()
        j = _Frames("upconv3x3", f"NB {NB} {H}x{W} C {C}->{Cout}", fam)
        for n in range(NB):
            img = out[n * 4 * H * W:(n + 1) * 4 * H * W].unflatten(0, (2 * H, 2 * W))
            for par in range(4):
                cols = conv_cols(x[n:n + 1], "ups", par=par).reshape(H * W, 4 * C)
                got = img[par >> 1::2, par & 1::2].reshape(H * W, Cout)
                _judge_linear(j, n, cols, got, w4[par * Cout:(par + 1) * Cout], b, what=f" parity {par}")
        fails.append(j.finish(_border_untouched(obuf, _INNER)))
        del xb, x, obuf, out
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


# ---- GEMMs
@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N,res,kind", GEMM_ROWS)
def test_gemm_rows_chunk_within_bound(ops, M, K, N, res, kind):
    """The 1x1 shortcuts and the mid-block q / k / to_out projections over all 16 frames (rows M = 16 HW)."""
    hw = M // CHUNK
    fails = []
    for fam in FAMS:
        seed = _seed(M, K, N, res, _FI[fam])
        _, _, w, b, _, _ = gemm_inputs(fam, _gen(seed, -1), 1, K, 0, N)
        abuf, a = _bordered(M, K)
        for n in range(CHUNK):
            a[n * hw:(n + 1) * hw] = _act_frame(fam, seed, n, hw, K)
        rbuf, r = _bordered(M, N) if res else (None, None)
        for n in range(CHUNK if res else 0):
            r[n * hw:(n + 1) * hw] = torch.randn(hw, N, device="cuda", generator=_gen(seed, CHUNK + n)).bfloat16()
        obuf, out = _bordered(M, N)
        ops.gemm(a, w, b, residual=r, out=out)
        torch.cuda.synchronize()
        j = _Frames(f"gemm {kind}", f"M {M} K {K} N {N}", fam)
        for n in range(CHUNK):
            sl = slice(n * hw, (n + 1) * hw)
            _judge_linear(j, n, a[sl], out[sl], w, b, None if r is None else r[sl])
        fails.append(j.finish(_border_untouched(obuf, _INNER)))
        del abuf, a, rbuf, r, obuf, out
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", ATTENTION)
def test_mid_attention_frame15_within_bound(ops, hw):
    """vae.py _attn on frame 15's row slice of 16-frame q / k / xn: scores (fp32, scale C^-1/2), softmax_rows,
    V^T = Wv xn^T (the activations as the W operand) and P V + bv into frame 15's rows of o; o's other frames untouched."""
    C, last = C_ATT, CHUNK - 1
    sl = slice(last * hw, CHUNK * hw)
    fails = []
    for fam in ("flat", "blocks"):
        seed = _seed(hw, C, _FI[fam])
        # q / xn: 64-wide channel blocks scaled 2^+-6 in the blocks family, k / Wv inversely (same products, wide operands)
        e = torch.exp2(_block_exp(C)).cuda() if fam == "blocks" else torch.ones(C, device="cuda")
        bufs = []
        for t, s in enumerate((e, 1 / e, e)):
            buf, v = _bordered(CHUNK * hw, C)
            for n in range(CHUNK):
                v[n * hw:(n + 1) * hw] = (_act_frame("flat", seed, 3 * n + t, hw, C).float() * s).bfloat16()
            bufs.append(buf)
        q, k, xn = (buf[_INNER] for buf in bufs)
        wv = (torch.randn(C, C, device="cuda", generator=_gen(seed, -1)) / math.sqrt(C) / e).bfloat16()
        bv = torch.randn(C, device="cuda", generator=_gen(seed, -2)).bfloat16().float()
        sbuf, scores = _bordered(hw, hw, torch.float32)
        pbuf, probs = _bordered(hw, hw)
        vbuf, vt = _bordered(C, hw)
        obuf, o = _bordered(CHUNK * hw, C)
        ops.gemm(q[sl], k[sl], scale=C ** -0.5, out=scores, out_f32=True)
        ops.softmax_rows(scores, out=probs)
        ops.gemm(wv, xn[sl], out=vt)
        ops.gemm(probs, vt, bv, out=o[sl])
        torch.cuda.synchronize()
        case = f"HW {hw} frame {last}"
        j = _Frames("attention scores", case, fam)
        for r0, r1 in _rows(hw, C, hw):
            ref, ref_abs, prod = linear_ref64(q[sl][r0:r1], k[sl], scale=C ** -0.5)
            j.add(last, scores[r0:r1], ref, linear_bound(ref, ref_abs, prod, C), bf16_out=False, what=f" rows {r0}..")
        fails.append(j.finish(_border_untouched(sbuf, _INNER)))
        j = _Frames("softmax_rows", case, fam)
        for r0, r1 in _rows(hw, 0, hw):
            ref, bnd = softmax_ref64(scores[r0:r1])
            j.add(last, probs[r0:r1], ref, bnd, what=f" rows {r0}..")
        fails.append(j.finish(_border_untouched(pbuf, _INNER)))
        j = _Frames("attention V^T", case, fam)
        _judge_linear(j, last, wv, vt, xn[sl])
        fails.append(j.finish(_border_untouched(vbuf, _INNER)))
        j = _Frames("attention P V", case, fam)
        _judge_linear(j, last, probs, o[sl], vt, bv)
        inner = (slice(3 + last * hw, 3 + CHUNK * hw), _INNER[1])
        fails.append(j.finish(_border_untouched(obuf, inner)))
        del bufs, q, k, xn, sbuf, scores, pbuf, probs, vbuf, vt, obuf, o
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


# ---- conv_in, conv_out_tc
@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,Cout", CONV_IN)
def test_conv_in_chunk_within_bound(ops, NB, H, W, Cout):
    """The decoder's conv_in with pre_scale = 1 / 0.18215 and the 4 x 4 post_quant_conv, on frames 1..16 of a buffer whose
    frames 0 and 17 are NaN."""
    fails = []
    for fam in ("flat", "frames"):
        seed = _seed(NB, H, Cout, _FI[fam])
        xb = torch.full((NB + 2, 4, H, W), float("nan"), device="cuda").bfloat16()
        for n in range(NB):
            xb[n + 1] = _act_frame(fam, seed, n, 4, H * W).view(4, H, W)
        x = xb[1:NB + 1]
        g = _gen(seed, -1)
        w = (torch.randn(Cout, 4, 3, 3, device="cuda", generator=g) / 6).bfloat16().float()
        b = torch.randn(Cout, device="cuda", generator=g).bfloat16().float()
        pre = (1 / SCALING, torch.randn(4, 4, device="cuda", generator=g).bfloat16().float(),
               torch.randn(4, device="cuda", generator=g).bfloat16().float())
        obuf, out = _bordered(NB * H * W, Cout)
        ops.conv_in(x, w.reshape(Cout, 36).t().contiguous(), b, Cout, out=out, pre_scale=pre[0], pre_w=pre[1],
                    pre_b=pre[2])
        torch.cuda.synchronize()
        j = _Frames("conv_in", f"NB {NB} {H}x{W} 4->{Cout}", fam)
        for n in range(NB):
            ref, bnd = _conv_in_ref64(x[n:n + 1], w, b, pre=pre)
            j.add(n, out[n * H * W:(n + 1) * H * W], ref, bnd)
        fails.append(j.finish(_border_untouched(obuf, _INNER)))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("NB,H,W,C,co", CONV_OUT)
def test_conv_out_tc_chunk_within_bound(ops, NB, H, W, C, co):
    """128 -> 3 with post = (v / 2 + 0.5).clamp(0, 1) into frames 16..31 of a sentinel-filled fp32 (3, 48, H, W) video,
    as VExpressPipeline.decode_latents passes its second chunk; the frames outside the view stay untouched."""
    hw = H * W
    fails = []
    for fam in FAMS:
        seed = _seed(NB, H, C, co, _FI[fam])
        w, _ = _conv_weights(fam, seed, C, co, 9)
        b = torch.randn(co, device="cuda", generator=_gen(seed, -2)).bfloat16().float()
        wp, bp = ops.pack_conv_out(w.view(co, 3, 3, C).permute(0, 3, 1, 2), b)
        xb, x = _nan_frames(fam, seed, NB, H, W, C)
        video = _sentinel_buf((co, 3 * NB, H, W), torch.float32)
        out = video[:, NB:2 * NB].permute(1, 0, 2, 3)
        ops.conv_out_tc(x.view(NB * hw, C), NB, H, W, wp, bp, out, post=True)
        torch.cuda.synchronize()
        j = _Frames("conv_out_tc", f"NB {NB} {H}x{W} C {C}->{co} post", fam)
        for n in range(NB):
            cols = conv_cols(x[n:n + 1]).reshape(hw, 9 * C)
            got = out[n].permute(1, 2, 0).reshape(hw, co)
            for r0, r1 in _rows(hw, 9 * C, wp.shape[0]):
                ref, ref_abs, prod = linear_ref64(cols[r0:r1], wp, bp)
                ref = ref[:, :co]
                bnd = 2.0 ** -8 * ref.abs() + linear_bound(ref, ref_abs[:, :co], prod[:, :co], 9 * C)  # bf16 conv output
                j.add(n, got[r0:r1], (0.5 * ref + 0.5).clamp(0, 1), 0.5 * bnd + 2.0 ** -22, bf16_out=False)
        rest = torch.cat([video[:, :NB], video[:, 2 * NB:]], 1)
        ok = bool((rest.view(torch.int32) == _SENTINEL32).all())
        fails.append(j.finish("" if ok else "frames outside the output view written"))
        del xb, x, video, out
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------- the composed decoder (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("h", LATENTS)
def test_vae_decode_chunk_vs_fp64(h):
    """16 distinct latent frames through AutoencoderKL.decode_latents into a (3, 16, H, W) video view; frames 0, 15 and
    those holding element or byte 2^31 of a decoder tensor against the oracle decoding that frame alone."""
    from oracle import vx_oracle as O
    from test_pipeline_gpu import build_vae
    from test_size768_bounds_gpu import _NET as NET768, _judge_taps, _oracle
    vcfg = O.VAE_CFG
    vsd = O.synth_state_dict(O.vae_param_shapes(vcfg), 1235)
    frames = sorted({0, CHUNK - 1} | set(_big_frames(h)))
    lat = SCALING * torch.randn(1, 4, CHUNK, h, h, generator=torch.Generator().manual_seed(80 + h))
    vae = build_vae(vcfg, vsd)
    video = torch.empty((3, CHUNK, 8 * h, 8 * h), device="cuda", dtype=torch.float32)
    z = lat[0].permute(1, 0, 2, 3).bfloat16().cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.time()
    vae.decode_latents(z, out=video.permute(1, 0, 2, 3))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    _NET.append(f"vae decode {CHUNK} x {h}x{h} -> {8 * h}x{8 * h}: {time.time() - t0:.2f} s (first call), peak device "
                f"memory {peak / 2 ** 30:.2f} GiB ({(peak - base) / 2 ** 30:.2f} GiB above the weights, latents and video)")
    print(_NET[-1])
    prod = {f"frame {n}": video[:, n].clone() for n in frames}
    assert torch.isfinite(video).all()
    del vae, video, z
    torch.cuda.empty_cache()
    res = {}
    for dt in (torch.float64, torch.bfloat16):
        sdd = {k: v.bfloat16().to(device="cuda", dtype=dt) for k, v in vsd.items()}
        res[dt] = {f"frame {n}": _oracle(O, O.decode_latents, sdd, vcfg,
                                         lat[:, :, n:n + 1].bfloat16().to(device="cuda", dtype=dt))[0, :, 0]
                   for n in frames}
        del sdd
    _judge_taps(f"vae decode chunk {h}x{h} frames {frames}", prod, res[torch.float64], res[torch.bfloat16], len(frames))
    _NET.append(NET768[-1])
