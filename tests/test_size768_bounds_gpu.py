"""The 768 x 768 configuration (96 x 96 latents) against fp64 references: the attention, audio and LayerNorm-fused GEMM
kernels at the shapes the engine issues there, then the composed UNet, ReferenceNet and VAE end to end.

1. Case list (CPU).  ``_RecordingOps`` (tests/test_host_cpu._ShapeOps, recording each call's shape-defining arguments)
   stands in for ``ops`` while ``UNetEngine.forward_frames`` and ``RefNetEngine.forward`` run at full width on the meta
   device: 96 x 96 latents, CFG with the reference bank (the uncond-zero shortcut and the full two-half form), f = 16,
   n = 1 and 2 samples, under the default, VX_LN_FOLD and VX_LN_FUSE modes.  Every recorded call must be covered by a GPU
   case of this file (``_case_keys``).  What "covered" means per family:
   * flash self-attention (kv_div = 1): same (Nq, Nk, heads, hd).  Query batch b reads kv batch b only; the cases run two
     batches, so a read across the batch edge meets the other batch's keys (family poison).
   * reference attention (kv_div > 1): the exact (Bq, Bkv, Nq, Nk, heads, hd, kv_div): the kv batch is b // kv_div.
   * temporal attention: same (f, HW, heads, hd); the clip count b only repeats independent (clip, pixel) items.
   * audio cross-attention: same (rows per frame, heads, hd, Lk); frames only repeat independent items.
   * GEMMs (gemm_ln, gemm_lnfold, gemm_lnparts, gemm_rowsums, and ops.gemm with GEGLU or a residual): same (K, N, GEGLU,
     residual, bias2 rows per frame) and the same rows per sample (M / n): an n-sample call is the one-sample call over
     n times the 128-row tiles.  The cases run the one-sample M (up to 2304 row tiles at M = 294912).  That normal form
     assumes the kernels' offsets do not overflow between the two: the two-sample operands at the 9216 level reach
     589824 x 2560 (ff1 before the GEGLU halving: under 2^31 elements, over 2^31 bytes), so PLAIN_N2 runs ff1 and ff2 at
     the two-sample M = 589824 as well.
   Every table entry must also cover a recorded call, so removing any entry makes ``test_engine_calls_at_768_are_covered``
   fail.  The 24-frame temporal cases (TEMPORAL_24, the pipeline's default context window) and gemm_ln (not wired into the
   engine) are checked beyond the recording.

2. Kernel cases (GPU), each judged by its sibling file's harness and bound, unchanged:
   tests/test_attention_bounds_gpu.py (_run_flash, _run_temporal, _run_smallkv), tests/test_lnfold_bounds_gpu.py
   (_run_paths: section 1 bound, and section 2 -- LayerNorm64 W^T under the default path's bound -- where it applies,
   _rowsums / _check_rowsums for the producer) and tests/test_gemm_bounds_gpu.py (linear_ref64 / geglu_ref64 +
   bound_check).  The plain GEMMs are judged one row chunk at a time against a reference of that chunk, so that the fp64
   temporaries of an M = 294912 output stay a few hundred MB.

3. The composed network (GPU), after tests/test_fullwidth_gpu.py: the reference is the oracle in fp64 on the GPU, the
   yardstick the same oracle in torch.bfloat16 on the GPU (what ``.to(bfloat16)`` does to the reference).  Every tap must
   satisfy e_prod <= 1.5 e_eager + 2e-3 (relative L2 against fp64), with no NaN / Inf and the tap count asserted.  The
   oracle's F.scaled_dot_product_attention would materialise 9216^2 fp64 score blocks per head; ``_oracle_sdpa_chunked``
   replaces the oracle's ``F`` for the duration of a case with a proxy whose fp64 SDPA is chunked over query rows.
"""
import math
import time

import pytest
import torch
import torch.nn.functional as F

from test_host_cpu import _ShapeOps, _cpu_engine

H768 = 96                                   # latent side of a 768 x 768 video
F768 = 16                                   # frames of the context window
LEVELS = [(320, 9216), (640, 2304), (1280, 576), (1280, 144)]     # (C, HW) of the four UNet levels at 96 x 96
HEADS = 8


# ---------------------------------------------------------------------------------------------------------- case tables
# flash self-attention: (Nq = Nk, hd); families flat, peaked, rising, poison at Bq = 2
FLASH_SELF = [(9216, 40), (2304, 80), (576, 160), (144, 160)]
# reference attention (attn1_5): (Bq, Bkv, Nk, hd, kv_div) with Nq = Nk.  Per level: CFG x 16 frames (kv_div 16, Bq 32),
# two samples (kv_div 32, Bq 64), and the uncond-zero shortcut (cond half only, Bkv 1) for one and two samples.
FLASH_REF = [(bq, bkv, n, hd, kv) for n, hd in FLASH_SELF
             for bq, bkv, kv in ((32, 2, 16), (64, 2, 32), (16, 1, 16), (32, 1, 32))]
# temporal attention: (f, HW, hd), b = 2 clips; the engine's 16-frame window (24 frames: TEMPORAL_24, beyond the recording)
TEMPORAL = [(F768, hw, c // HEADS) for c, hw in LEVELS]
TEMPORAL_24 = [(24, hw, c // HEADS) for c, hw in LEVELS]
# audio cross-attention: (frames, rows per frame, hd, Lk): the UNet's 5 audio tokens and the ReferenceNet's one zero token
SMALLKV = [(32, hw, c // HEADS, 5) for c, hw in LEVELS] + [(4, hw, c // HEADS, 1) for c, hw in LEVELS]
# LayerNorm-fused GEMMs at the one-sample engine M = 2 x 16 x HW: (K, HW, kind); kind qkv is the attn1 projection, qkv_pe
# the motion projection (the positional encoding enters as a per-frame bias2, rows_per_frame = HW), to_q the attn1_5 /
# attn2 query, geglu the feed-forward's first GEMM
LN_GEMMS = [(c, hw, kind) for c, hw in LEVELS for kind in ("qkv", "qkv_pe", "to_q", "geglu")]
LN_N = {"qkv": 3, "qkv_pe": 3, "to_q": 1, "geglu": 8}
# producers of the statistics hand-over (VX_LN_FUSE): (K = N, HW, residual): proj_in, and the attention to_out
ROWSUMS = [(c, hw, res) for c, hw in LEVELS for res in (False, True)]
# plain GEMMs with GEGLU or a residual: (C, rows, kind): the UNet's at rows = 2 x 16 x HW, the ReferenceNet's at HW;
# kind geglu is ff1 (N = 8C), residual the to_out / proj_out (C x C, output scaled), ff2 the feed-forward's second GEMM
PLAIN = [(c, m, kind) for c, hw in LEVELS for m in (2 * F768 * hw, hw) for kind in ("geglu", "residual", "ff2")]
# the same at the two-sample rows of the 9216 level (beyond the normal form: the largest operands of the file)
PLAIN_N2 = [(320, 4 * F768 * 9216, kind) for kind in ("geglu", "ff2")]


def _plain_shape(C, kind):
    """(K, N) of a PLAIN kind at width C (N before the GEGLU halving)."""
    return (4 * C, C) if kind == "ff2" else (C, 8 * C if kind == "geglu" else C)


def _case_keys():
    """{call key (the normal form of ``_call_key``) -> the table entry that covers it}; one key per entry, except that
    an LN_GEMMS entry stands for its gemm_lnfold, gemm_lnparts and (K <= 512) gemm_ln calls."""
    keys = {}

    def add(key, entry):
        assert key not in keys, (key, entry, keys[key])
        keys[key] = entry
    for n, hd in FLASH_SELF:
        add(("flash", None, None, n, n, HEADS, hd, 1), ("FLASH_SELF", n, hd))
    for bq, bkv, n, hd, kv in FLASH_REF:
        add(("flash", bq, bkv, n, n, HEADS, hd, kv), ("FLASH_REF", bq, bkv, n, hd, kv))
    for f, hw, hd in TEMPORAL:
        add(("temporal", f, hw, HEADS, hd), ("TEMPORAL", f, hw, hd))
    for fr, hw, hd, lk in SMALLKV:
        add(("smallkv", hw, HEADS, hd, lk), ("SMALLKV", fr, hw, hd, lk))
    for c, hw, kind in LN_GEMMS:
        div = hw if kind == "qkv_pe" else 0
        for op in ("gemm_lnfold", "gemm_lnparts") + (("gemm_ln",) if c <= 512 else ()):
            add((op, c, LN_N[kind] * c, kind == "geglu", False, div, 2 * F768 * hw), ("LN_GEMMS", c, hw, kind))
    for c, hw, res in ROWSUMS:
        add(("gemm_rowsums", c, c, False, res, 0, 2 * F768 * hw), ("ROWSUMS", c, hw, res))
    for c, m, kind in PLAIN:
        K, N = _plain_shape(c, kind)
        add(("gemm", K, N, kind == "geglu", kind != "geglu", 0, m), ("PLAIN", c, m, kind))
    return keys


def _call_key(op, a, k, n):
    """The normal form of one ops call of an n-sample forward (module docstring, section 1), or None for ops outside this
    file's families."""
    if op == "flash_attention":
        q, kk = a[0], a[1]
        heads, Nq, Nk = a[3], a[4], a[5]
        kv_div = a[6] if len(a) > 6 else k.get("kv_div", 1)
        Bq, Bkv = q.shape[0] // Nq, kk.shape[0] // Nk
        assert Bq * Nq == q.shape[0] and Bkv * Nk == kk.shape[0]
        if kv_div == 1:
            assert Bkv == Bq
            return ("flash", None, None, Nq, Nk, heads, q.shape[1] // heads, 1)
        return ("flash", Bq, Bkv, Nq, Nk, heads, q.shape[1] // heads, kv_div)
    if op == "temporal_attention":
        q, b, f, HW, heads = a[0], a[3], a[4], a[5], a[6]
        assert q.shape[0] == b * f * HW
        return ("temporal", f, HW, heads, q.shape[1] // heads)
    if op == "smallkv_attention":
        q, rpf, heads, Lk = a[0], a[3], a[4], a[5]
        assert q.shape[0] % rpf == 0 and a[1].shape[0] == q.shape[0] // rpf * Lk
        return ("smallkv", rpf, heads, q.shape[1] // heads, Lk)
    if op in ("gemm_ln", "gemm_lnfold", "gemm_lnparts", "gemm_rowsums", "gemm"):
        x, w = a[0], a[1]
        geglu, res = bool(k.get("geglu")), k.get("residual") is not None
        if op == "gemm" and not (geglu or res):
            return None
        assert k.get("a2") is None and x.shape[0] % n == 0
        div = k.get("bias2_div", 1) if k.get("bias2") is not None else 0
        return (op, x.shape[1], w.shape[0], geglu, res, div, x.shape[0] // n)
    return None


class _RecordingOps(_ShapeOps):
    """_ShapeOps that also records the normal form of every call (``_call_key``) with the first shapes that produced it."""

    def __init__(self):
        super().__init__()
        self.seen = {}
        self.n = 1                  # samples of the forward being recorded

    def __getattr__(self, op):
        run = super().__getattr__(op)

        def rec(*a, **k):
            key = _call_key(op, a, k, self.n)
            if key is not None:
                self.seen.setdefault(key, (op, [tuple(t.shape) for t in a if torch.is_tensor(t)]))
            return run(*a, **k)
        return rec


def _record_engine_calls(monkeypatch):
    """Run the full-width engines at 96 x 96 on the meta device under every mode and form -> {key: (op, shapes)}."""
    from oracle import vx_oracle as O
    from test_unet_gpu import UNET_EXTRA
    from vexpress_b200.modules import ReferenceAttentionControl, UNet2DConditionModel, UNet3DConditionModel
    from vexpress_b200.modules import unet_2d_condition, unet_3d
    cfg = O.DEFAULT_CFG
    h, f = H768, F768
    with torch.device("meta"):
        m = UNet3DConditionModel(block_out_channels=cfg["block_out_channels"],
                                 cross_attention_dim=cfg["cross_attention_dim"], **UNET_EXTRA).to(torch.bfloat16)
        net = UNet2DConditionModel(block_out_channels=cfg["block_out_channels"],
                                   cross_attention_dim=cfg["cross_attention_dim"]).to(torch.bfloat16)
        engines = []
        for fold, fuse in (("0", "0"), ("1", "0"), ("0", "1")):
            monkeypatch.setenv("VX_LN_FOLD", fold)
            monkeypatch.setenv("VX_LN_FUSE", fuse)
            eng = _cpu_engine(unet_3d.UNetEngine, m, "meta")
            assert (eng.ln_fold, eng.ln_fuse) == (fold == "1", fuse == "1")
            engines.append(eng)
        ReferenceAttentionControl(net, mode="write", fusion_blocks="full", do_classifier_free_guidance=True)
        reng = _cpu_engine(unet_2d_condition.RefNetEngine, net, "meta")
        fake = _RecordingOps()
        monkeypatch.setattr(unet_3d, "ops", fake)
        monkeypatch.setattr(unet_2d_condition, "ops", fake)
        for eng in engines:
            for uncond_zero in (True, False):
                # the bank K / V of one block: [uncond | cond] x the level's h x w tokens
                eng._bank_kv = lambda name, block, e=eng, z=uncond_zero: (
                    torch.empty(2 * _bank_rows(name, h), 2 * e.W[name + ".norm1.weight"].shape[0]), z)
                for n in (1, 2):
                    fake.n = n
                    b = 2 * n
                    frames = torch.empty(b * f, 4, h, h, dtype=torch.bfloat16)
                    enc = torch.empty(b * f, 5, cfg["cross_attention_dim"])
                    kps = torch.empty(b * f * h * h, cfg["block_out_channels"][0], dtype=torch.bfloat16)
                    out = eng.forward_frames(frames, 499, enc, kps, None, 2, f, n=n)
                    assert out.shape == (b * f, 4, h, h)
        fake.n = 1
        rout = reng.forward(torch.empty(1, 4, h, h, dtype=torch.bfloat16), 0, torch.empty(1, 1, cfg["cross_attention_dim"]))
        assert rout.shape == (1, 4, h, h)
    return fake.seen


def _bank_rows(name, h):
    """Tokens of the ReferenceNet bank a reader block reads: its level's h x w."""
    if name.startswith("down_blocks."):
        s = int(name.split(".")[1])
    elif name.startswith("up_blocks."):
        s = 3 - int(name.split(".")[1])
    else:
        s = 3
    return (h >> s) ** 2


def test_engine_calls_at_768_are_covered(monkeypatch):
    """Every attention and LayerNorm-fused / GEGLU / residual GEMM call of the 96 x 96 engines has a GPU case here, and
    every case-table entry covers a call the engines make (so removing any entry fails)."""
    seen = _record_engine_calls(monkeypatch)
    cases = _case_keys()
    for k in sorted(seen, key=str):
        print(("   " if k in cases else "!! ") + str(k))
    missing = {k: v for k, v in seen.items() if k not in cases}
    assert not missing, "engine calls without a GPU case:\n" + "\n".join(f"{k}: {v}" for k, v in missing.items())
    used = {cases[k] for k in seen}
    stale = set(cases.values()) - used
    assert not stale, f"case-table entries no engine call needs: {sorted(stale, key=str)}"
    beyond = sorted((k for k in cases if k not in seen), key=str)
    print(f"{len(seen)} call forms recorded, all covered by {len(used)} table entries; keys beyond the engine's: {beyond}")


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture(scope="module", autouse=True)
def _time_and_memory():
    """Prints the file's GPU wall time and peak device memory, and each family's worst bound ratio, at the end."""
    import test_attention_bounds_gpu as A
    import test_lnfold_bounds_gpu as L
    t0 = time.time()
    yield
    for name, table in (("attention", A._WORST), ("lnfold", L._WORST), ("gemm", _WORST)):
        for path, (worst, case) in sorted(table.items()):
            print(f"worst bound ratio [{name}] {path:18s} {worst:.3f}  ({case})")
    for row in _NET:
        print(row)
    if _PEAK:
        top = sorted(_PEAK.items(), key=lambda kv: -kv[1])
        print(f"size768 file: {time.time() - t0:.1f} s, peak device memory {top[0][1]:.2f} GiB ({top[0][0]}); next: "
              + ", ".join(f"{n} {v:.2f}" for n, v in top[1:6]))


PEAK_GIB = 40.0              # the file shares its GPU: no case may hold more than this at once
_PEAK = {}                   # case -> peak device memory (GiB) allocated while it ran


@pytest.fixture(autouse=True)
def _case_peak(request):
    """Peak device memory of each GPU case, printed at the end of the file and held under PEAK_GIB."""
    if request.node.get_closest_marker("gpu") is None or not torch.cuda.is_available():
        yield
        return
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    _PEAK[request.node.name] = peak
    assert peak <= PEAK_GIB, f"{request.node.name}: peak device memory {peak:.2f} GiB"


_WORST = {}                  # plain GEMM kind -> (worst ratio, case)
_NET = []                    # network summary lines
ATT_FAMILIES = ("flat", "peaked", "rising", "poison")


@pytest.mark.gpu
@pytest.mark.parametrize("n,hd", FLASH_SELF)
def test_flash_self_attention_768_within_bound(ops, n, hd):
    from test_attention_bounds_gpu import _run_flash
    _run_flash(ops, ATT_FAMILIES, 2, n, n, HEADS, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("bq,bkv,n,hd,kv_div", FLASH_REF)
def test_reference_attention_768_within_bound(ops, bq, bkv, n, hd, kv_div):
    """attn1_5 over the bank: query batch b reads bank block b // kv_div (poison sits in block 1)."""
    from test_attention_bounds_gpu import _run_flash
    assert (bq + kv_div - 1) // kv_div == bkv
    _run_flash(ops, ("flat", "rising", "poison"), bq, n, n, HEADS, hd, kv_div)


@pytest.mark.gpu
@pytest.mark.parametrize("f,hw,hd", TEMPORAL + TEMPORAL_24)
def test_temporal_attention_768_within_bound(ops, f, hw, hd):
    from test_attention_bounds_gpu import _run_temporal
    _run_temporal(ops, ("flat", "peaked", "poison"), 2, f, hw, HEADS, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("frames,rpf,hd,lk", SMALLKV)
def test_audio_attention_768_within_bound(ops, frames, rpf, hd, lk):
    from test_attention_bounds_gpu import _run_smallkv
    _run_smallkv(ops, ("flat", "peaked", "poison"), frames, rpf, HEADS, hd, lk)


@pytest.mark.gpu
@pytest.mark.parametrize("c,hw,kind", LN_GEMMS)
def test_layernorm_gemms_768_within_bound(ops, c, hw, kind):
    """lnfold, lnparts (with its gemm_rowsums producer) and gemm_ln (K <= 512) at M = 2 x 16 x HW; section 2 of
    test_lnfold_bounds_gpu (against LayerNorm64 W^T) where it applies and the fp64 temporaries stay under 1.25 GB each."""
    from test_lnfold_bounds_gpu import ALL_PATHS, _run_paths
    M, N = 2 * F768 * hw, LN_N[kind] * c
    paths = ALL_PATHS if c <= 512 else ALL_PATHS[:2]
    geglu = kind == "geglu"
    parity = M * (N // 2 if geglu else N) * 8 <= 1.25 * 2 ** 30
    bad = []
    for fam in ("flat", "offset"):
        bad += _run_paths(ops, paths, fam, M, c, N, geglu=geglu, div=hw if kind == "qkv_pe" else 0, tag=f" {kind}",
                          parity=parity)
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("c,hw,res", ROWSUMS)
def test_rowsums_producer_768(ops, c, hw, res):
    """gemm_rowsums as the engine calls it (K = N = C, with and without the residual): the output bits of ops.gemm, every
    slot within its bound of the fp64 sums of those bits, nothing written past nparts or M."""
    from test_gemm_bounds_gpu import _INNER, _border_untouched, _in_nan
    from test_lnfold_bounds_gpu import _check_rowsums, _rowsums
    M = 2 * F768 * hw
    g = torch.Generator(device="cuda").manual_seed(M + c + res)
    a = torch.randn(M, c, device="cuda", generator=g).bfloat16()
    w = (torch.randn(c, c, device="cuda", generator=g) / math.sqrt(c)).bfloat16()
    b = (0.5 * torch.randn(c, device="cuda", generator=g)).bfloat16().float()
    r = torch.randn(M, c, device="cuda", generator=g).bfloat16() if res else None
    h, hbuf, pbuf, nparts = _rowsums(ops, _in_nan(a), _in_nan(w), b, _in_nan(r), M, c)
    twin = ops.gemm(a, w, b, residual=r)
    bad = _check_rowsums(ops, h, pbuf, nparts, M, c, twin)
    border = _border_untouched(hbuf, _INNER)
    print(f"rowsums M {M} K = N {c} res {res}: nparts {nparts}, " + ("; ".join(bad + [border]) or "ok"))
    assert not bad and not border, (bad, border)


@pytest.mark.gpu
@pytest.mark.parametrize("c,m,kind", PLAIN + PLAIN_N2)
def test_plain_gemms_768_within_bound(ops, c, m, kind):
    """ff1 (GEGLU epilogue), to_out / proj_out (scaled, + residual) and ff2 (+ residual) at the engine's rows, judged one row
    chunk at a time by test_gemm_bounds_gpu's references and bound_check."""
    from test_gemm_bounds_gpu import (_INNER, _border_untouched, _bordered, _chunks, _in_nan, bound_check, geglu_ref64,
                                      linear_bound, linear_ref64)
    K, N = _plain_shape(c, kind)
    g = torch.Generator(device="cuda").manual_seed(m * 7 + K + N)
    a = torch.randn(m, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    b = (0.5 * torch.randn(N, device="cuda", generator=g)).bfloat16().float()
    geglu = kind == "geglu"
    scale = 0.95 if kind == "residual" else 1.0
    res = None if geglu else torch.randn(m, N, device="cuda", generator=g).bfloat16()
    obuf, out = _bordered(m, N // 2 if geglu else N)
    if geglu:
        wp, bp, _ = ops.pack_geglu(w, b)
        ops.gemm(_in_nan(a), _in_nan(wp), bp, geglu=True, out=out)
    else:
        ops.gemm(_in_nan(a), _in_nan(w), b, scale=scale, residual=_in_nan(res), out=out)
    torch.cuda.synchronize()
    worst, where, err2, ref2 = 0.0, "", 0.0, 0.0
    for r0, r1 in _chunks(m, K, 4 * N):
        if geglu:
            ref, bnd = geglu_ref64(a[r0:r1], w, b)
        else:
            ref, ref_abs, prod_abs = linear_ref64(a[r0:r1], w, b, scale=scale, residual=res[r0:r1])
            bnd = linear_bound(ref, ref_abs, prod_abs, K)
        wst, _, wh = bound_check(out[r0:r1], ref, bnd)
        if wst > worst or not where:
            worst, where = wst, f"rows {r0}..{r1}: {wh}"
        err2 += float((out[r0:r1].double() - ref).norm()) ** 2
        ref2 += float((ref if geglu else ref - res[r0:r1].double()).norm()) ** 2
    rel = math.sqrt(err2 / ref2)
    case = f"M {m} K {K} N {N} {kind}"
    print(f"gemm {case}: worst ratio {worst:.3f}, rel {rel:.2e}")
    if worst > _WORST.get(kind, (-1.0, ""))[0]:
        _WORST[kind] = (worst, case)
    border = _border_untouched(obuf, _INNER)
    assert worst <= 1 and rel < 5e-3 and not border and not torch.isnan(out.float()).any(), (case, where, rel, border)


# ------------------------------------------------------------------------------------------- the composed network (GPU)
REF_W, AUDIO_W = 0.95, 3.0


class _ChunkedSDPA:
    """Stands in for the oracle's ``F``: everything is torch.nn.functional, except that an fp64
    scaled_dot_product_attention is computed over query-row chunks whose score block stays under 256 MB."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def scaled_dot_product_attention(q, k, v, *args, **kw):
        if q.dtype != torch.float64 or args or kw:
            return F.scaled_dot_product_attention(q, k, v, *args, **kw)
        Lq, Lk = q.shape[-2], k.shape[-2]
        out = torch.empty(q.shape[:-1] + (v.shape[-1],), dtype=q.dtype, device=q.device)
        rows = max(1, (256 << 20) // (8 * Lk * math.prod(q.shape[:-2])))
        kt = k.transpose(-1, -2) / math.sqrt(q.shape[-1])
        for r0 in range(0, Lq, rows):
            out[..., r0:r0 + rows, :] = torch.softmax(q[..., r0:r0 + rows, :] @ kt, -1) @ v
        return out


def _rel64(a, ref):
    ref = ref.double()
    return float((a.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _judge_taps(name, prod, fp64, eager, count):
    """Each tap: e_prod <= 1.5 e_eager + 2e-3 against fp64, finite -> prints every pair and the worst tap."""
    bad, worst = [], (0.0, "")
    keys = [k for k in fp64 if k in prod]
    for k in keys:
        e_p, e_e = _rel64(prod[k], fp64[k]), _rel64(eager[k], fp64[k])
        ratio = e_p / (1.5 * e_e + 2e-3)
        print(f"{name} tap {k:36s} e_prod {e_p:.3e}  e_eager {e_e:.3e}  ({ratio:.2f} of the limit)")
        if ratio > worst[0]:
            worst = (ratio, f"{k}: e_prod {e_p:.3e} e_eager {e_e:.3e}")
        if not torch.isfinite(prod[k]).all():
            bad.append(f"{k}: NaN or Inf")
        if not ratio <= 1:
            bad.append(f"{k}: e_prod {e_p:.3e} > 1.5 e_eager {e_e:.3e} + 2e-3")
    _NET.append(f"{name}: {len(keys)} taps, worst at {worst[0]:.2f} of the limit ({worst[1]})")
    print(_NET[-1])
    assert len(keys) == count, (name, len(keys), count)
    assert not bad, f"{name}:\n" + "\n".join(bad)


def _oracle(O, fn, *args, **kw):
    """An oracle call on the GPU (its own tensors are created there too) with the chunked fp64 attention."""
    with pytest.MonkeyPatch.context() as mp, torch.device("cuda"), torch.no_grad():
        mp.setattr(O, "F", _ChunkedSDPA())
        return fn(*args, **kw)


class _Taps32(dict):
    """A taps dict that keeps fp64 activations as fp32 (their rounding, 2^-24 relative, is far below every error judged
    here): the fp64 taps of a 64 x 64, 16-frame forward would otherwise hold about 15 GB."""

    def __setitem__(self, k, v):
        super().__setitem__(k, v.float() if v.dtype == torch.float64 else v)


@pytest.fixture(scope="module")
def unet768():
    """The product UNet on the GPU and the synthetic fp32 weights on the host; each case moves the fp64 and the bf16
    oracle weights to the GPU for its own oracle pass only."""
    from oracle import vx_oracle as O
    from test_unet_gpu import build_product
    cfg = O.DEFAULT_CFG
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
    lat, kps, audio, banks = O.synth_inputs(cfg, 4, H768, H768, True, 42)
    model, reader = build_product(cfg, sd, [b[1:] for b in banks], REF_W, AUDIO_W)
    yield dict(O=O, cfg=cfg, model=model, reader=reader, sd=sd)
    reader.clear()


UNET_TAPS = 63      # conv_in, 25 down, mid_block, 36 up (tests/test_fullwidth_gpu.py's block boundaries)


@pytest.mark.gpu
@pytest.mark.parametrize("h,f", [(H768, 4), (64, 16)])
def test_unet_fullwidth_every_tap_vs_fp64(unet768, h, f):
    """The full-width UNet with CFG and the bank: 96 x 96 latents at f = 4, and 64 x 64 at the bench window f = 16."""
    from test_unet_gpu import _Writer
    U = unet768
    O, cfg, model = U["O"], U["cfg"], U["model"]
    lat, kps, audio, banks = O.synth_inputs(cfg, f, h, h, True, 42)
    U["reader"].update(_Writer([b[1:].cuda() for b in banks]), True, dtype=torch.bfloat16)
    x = lat.repeat(2, 1, 1, 1, 1)
    enc = audio.reshape(-1, 5, cfg["cross_attention_dim"])
    t0 = time.time()
    d64 = lambda t: t.bfloat16().double().cuda()
    d16 = lambda t: t.bfloat16().cuda()
    taps64, taps16 = _Taps32(), {}
    sdd = {k: d64(v) for k, v in U["sd"].items()}
    ref = _oracle(O, O.unet_forward, sdd, cfg, d64(x), 499, d64(enc), d64(kps), [d64(b) for b in banks], REF_W,
                  AUDIO_W, taps=taps64)
    del sdd
    t1 = time.time()
    sdd = {k: d16(v) for k, v in U["sd"].items()}
    eager = _oracle(O, O.unet_forward, sdd, cfg, d16(x), 499, d16(enc), d16(kps), [d16(b) for b in banks], REF_W,
                    AUDIO_W, taps=taps16)
    del sdd
    t2 = time.time()
    eng = model.engine()
    b = x.shape[0]
    frames = x.bfloat16().cuda().permute(0, 2, 1, 3, 4).reshape(b * f, 4, h, h).contiguous()
    kps_nhwc = kps.bfloat16().cuda().permute(0, 2, 3, 4, 1).reshape(b * f * h * h, -1).contiguous()
    tapsp = {}
    out = eng.forward_frames(frames, 499, enc.cuda(), kps_nhwc, None, b, f, taps=tapsp)
    torch.cuda.synchronize()
    print(f"unet {h}x{h} f {f}: oracle fp64 {t1 - t0:.1f} s, bf16 eager {t2 - t1:.1f} s, product {time.time() - t2:.1f} s")
    tapsp["out"] = out.view(b, f, -1, h, h).permute(0, 2, 1, 3, 4)
    taps64["out"], taps16["out"] = ref, eager
    _judge_taps(f"unet {h}x{h} f={f}", tapsp, taps64, taps16, UNET_TAPS + 1)


@pytest.mark.gpu
def test_refnet_write_pass_vs_fp64():
    """The ReferenceNet write pass at 96 x 96: each of the 16 bank tensors and the output."""
    from oracle import vx_oracle as O
    from vexpress_b200.modules import ReferenceAttentionControl, UNet2DConditionModel
    from vexpress_b200.modules.unet_2d_condition import writer_block_names
    cfg = O.DEFAULT_CFG
    sd = O.synth_state_dict(O.refnet_param_shapes(cfg), 4321)
    net = UNet2DConditionModel(block_out_channels=cfg["block_out_channels"], cross_attention_dim=cfg["cross_attention_dim"])
    net.load_state_dict(sd, strict=True)
    net = net.to(torch.bfloat16).to("cuda")
    writer = ReferenceAttentionControl(net, do_classifier_free_guidance=True, mode="write", batch_size=1,
                                       fusion_blocks="full")
    x = torch.randn(1, 4, H768, H768, generator=torch.Generator().manual_seed(77))
    enc = torch.zeros(1, 1, cfg["cross_attention_dim"], device="cuda", dtype=torch.bfloat16)
    out = net(x.bfloat16().cuda(), timestep=0, encoder_hidden_states=enc, return_dict=False)[0]
    torch.cuda.synchronize()
    prod = {n[:-len(".transformer_blocks.0")]: blk.bank[0] for n, blk in zip(writer_block_names(), net.writer_blocks())}
    prod["out"] = out
    res = {}
    for dt in (torch.float64, torch.bfloat16):
        sdd = {k: v.bfloat16().to(device="cuda", dtype=dt) for k, v in sd.items()}
        banks, o = _oracle(O, O.refnet_forward, sdd, cfg, x.bfloat16().to(device="cuda", dtype=dt))
        res[dt] = dict(zip(O.bank_order(cfg), banks), out=o)
        del sdd
    writer.clear()
    _judge_taps("refnet 96x96", prod, res[torch.float64], res[torch.bfloat16], 17)


@pytest.mark.gpu
def test_vae_decode_768_vs_fp64():
    """The full-width VAE decoder (512/512/256/128): two 96 x 96 latent frames to 768 x 768, with the (x / 2 + 0.5) clamp."""
    from oracle import vx_oracle as O
    from test_pipeline_gpu import build_vae
    vcfg = O.VAE_CFG
    vsd = O.synth_state_dict(O.vae_param_shapes(vcfg), 1235)
    vae = build_vae(vcfg, vsd)
    lat = 0.18215 * torch.randn(1, 4, 2, H768, H768, generator=torch.Generator().manual_seed(78))
    out = vae.decode_latents(lat[0].permute(1, 0, 2, 3).bfloat16().cuda())
    torch.cuda.synchronize()
    res = {}
    for dt in (torch.float64, torch.bfloat16):
        sdd = {k: v.bfloat16().to(device="cuda", dtype=dt) for k, v in vsd.items()}
        res[dt] = {"video": _oracle(O, O.decode_latents, sdd, vcfg, lat.bfloat16().to(device="cuda", dtype=dt))[0]
                   .permute(1, 0, 2, 3)}
        del sdd
    assert out.shape == (2, 3, 768, 768)
    _judge_taps("vae decode 96x96 -> 768x768", {"video": out}, res[torch.float64], res[torch.bfloat16], 1)
