"""Every attention kernel against an fp64 reference, element by element, under an error bound a correct kernel cannot
exceed, on score distributions chosen to exercise the online softmax (running max, alpha, l, key-tail mask).

The bound, for every output element (``attention_ref64`` gives ``ref = P V`` and ``ref_abs = P |V|``, P the exact
softmax of the bf16 inputs):

    |out - ref| <= 2^-8 (ref_abs + |ref|) + Nk 2^-22 ref_abs

* The flash and the mma kernels round P to bf16 before P V.  That moves each term p_i v_i by at most u = 2^-8 of itself
  (round to nearest, 8 significant bits), so the sum by at most 2^-8 sum p_i |v_i| = 2^-8 ref_abs.  The normaliser l is
  summed from the unrounded P, so no second rounding enters through it.
* Rounding the output to bf16 adds at most 2^-8 |out|, taken as 2^-8 |ref| (the difference is second order).
* The last term covers fp32 accumulation of Nk products: Nk 2^-24 ref_abs, times 2 for tensor-core accumulation that may
  truncate instead of round, times 2 for the O / l division and the exponentials.
A correct kernel stays below the bound on any input, so a ratio above 1 is a bug, not a tolerance to widen.  The global
relative criterion ||out - ref|| / ||ref|| < 4e-3 of tests/test_ops_gpu.py is kept on every case as well: a key dropped
from a flat softmax over thousands of keys moves each element by less than the bound but moves the norm by more.

The data families (``family_inputs``) are functions of a torch.Generator, so the CPU self-test and the GPU cases run the
same code.  ``test_bound_rejects_injected_faults`` runs a torch model of the 64-key flash loop with injectable faults
through the same check: it is the evidence that the GPU cases would catch those faults in a kernel.
"""
import math
import os

import pytest
import torch

LOG2E = 1.4426950408889634
FAMILIES = ("flat", "peaked", "rising", "falling", "tail", "poison", "degenerate")
STEP = 64                      # keys per step of the flash loops
_SENTINEL = 0x7FC1             # a bf16 NaN no kernel produces: cells around an output slice hold it
_WORST = {}                    # kernel -> (worst bound ratio, case), printed at the end of the module


# ---------------------------------------------------------------------------------------------------------- reference
def attention_ref64(q, k, v, heads, Nq, Nk, kv_div=1, budget=256 << 20):
    """fp64 softmax(Q K^T / sqrt(hd)) V of bf16 token matrices q [Bq*Nq, C], k / v [Bkv*Nk, C] (kv batch of query batch
    b is b // kv_div) -> (ref, ref_abs) float64 [Bq*Nq, C]: P V and P |V|.  Batches and query rows are chunked so that
    no score block exceeds ``budget`` bytes."""
    C = q.shape[1]
    hd = C // heads
    Bq, Bkv = q.shape[0] // Nq, k.shape[0] // Nk
    split = lambda t, B, N: t.double().reshape(B, N, heads, hd).transpose(1, 2)      # (B, heads, N, hd)
    qd, kd, vd = split(q, Bq, Nq), split(k, Bkv, Nk), split(v, Bkv, Nk)
    ref = torch.empty((Bq, heads, Nq, hd), dtype=torch.float64, device=q.device)
    ref_abs = torch.empty_like(ref)
    per_row = heads * Nk * 8
    nb = max(1, budget // (per_row * Nq))
    rows = Nq if nb > 1 else max(1, budget // per_row)
    for b0 in range(0, Bq, nb):
        b1 = min(Bq, b0 + nb)
        kv = torch.arange(b0, b1, device=q.device) // kv_div
        kb, vb = kd[kv], vd[kv]
        for r0 in range(0, Nq, rows):
            r1 = min(Nq, r0 + rows)
            p = torch.softmax(qd[b0:b1, :, r0:r1] @ kb.transpose(-1, -2) / math.sqrt(hd), -1)
            ref[b0:b1, :, r0:r1] = p @ vb
            ref_abs[b0:b1, :, r0:r1] = p @ vb.abs()
    back = lambda t: t.transpose(1, 2).reshape(Bq * Nq, C)
    return back(ref), back(ref_abs)


def bound_check(out, ref, ref_abs, Nk, Nq, heads):
    """(worst ratio |out - ref| / bound, global relative error, description of the worst element).  NaN counts as an
    infinite ratio."""
    o = out.double().reshape(ref.shape)
    err = (o - ref).abs()
    bound = 2.0 ** -8 * (ref_abs + ref.abs()) + Nk * 2.0 ** -22 * ref_abs
    ratio = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / bound), nan=math.inf)
    i = int(ratio.argmax())
    row, col = divmod(i, ref.shape[1])
    hd = ref.shape[1] // heads
    worst = float(ratio.view(-1)[i])
    rel = float((o - ref).norm() / ref.norm())
    where = (f"worst at (batch {row // Nq}, row {row % Nq}, head {col // hd}, column {col % hd}): "
             f"out {float(o.view(-1)[i]):.6g} ref {float(ref.view(-1)[i]):.6g} ratio {worst:.3f}")
    return worst, rel, where


# ------------------------------------------------------------------------------------------------------- data families
def family_inputs(name, g, Bq, Nq, Bkv, Nk, heads, hd, poison_from=1, n_poison=16):
    """bf16 q [Bq*Nq, heads*hd], k / v [Bkv*Nk, heads*hd] on g's device.  u is one unit direction per head.
    flat       : N(0, 1).
    peaked     : Q, K x 3 -- scores spread over tens of log2 units, most exponentials underflow, alpha << 1 when the max
                 moves.
    rising     : Q leans on u, K climbs along u by 4 nats (at q.u = 3) per 64-key step for 12 steps: every step raises
                 the running max.
    falling    : the mirror image: the max is in step 0, every later alpha is 1.
    tail       : Q leans on u, one of the last four keys of every kv batch gets +12 nats: the dominant key sits in the
                 (partial) last step.
    poison     : keys [0, n_poison) of kv batches >= poison_from get scores ~16 nats above the rest and V x 30.  These are
                 real keys of their batch, placed where a kernel that reads past its own batch (the rows behind Nk, the
                 next item's frames or tokens) would pick them up.
    degenerate : heads cycle through Q = 0, identical K rows (both: uniform softmax) and K drawn from three prototypes
                 (tied maxima)."""
    dev = g.device
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    q, k, v = rn(Bq, Nq, heads, hd), rn(Bkv, Nk, heads, hd), rn(Bkv, Nk, heads, hd)
    u = rn(heads, hd)
    u = u / u.norm(dim=-1, keepdim=True)
    rt = math.sqrt(hd)
    if name == "peaked":
        q, k = 3 * q, 3 * k
    elif name in ("rising", "falling"):
        steps = (torch.arange(Nk, device=dev) // STEP).clamp(max=12).float()
        r = (4.0 * rt / 3) * (steps if name == "rising" else -steps)
        q = q + 3 * u
        k = k + r[None, :, None, None] * u
    elif name == "tail":
        q = q + 2 * u
        pos = Nk - 1 - torch.randint(0, min(4, Nk), (Bkv,), device=dev, generator=g)
        k[torch.arange(Bkv, device=dev), pos] += 6 * rt * u
    elif name == "poison":
        q = q + 2 * u
        mask = torch.zeros(Bkv, Nk, dtype=torch.bool, device=dev)
        mask[poison_from:, :n_poison] = True
        k[mask] += 8 * rt * u
        v[mask] *= 30
    elif name == "degenerate":
        sel = torch.arange(heads, device=dev) % 3
        q[:, :, sel == 0] = 0
        k[:, :, sel == 1] = k[:, :1, sel == 1]
        proto = torch.randint(0, min(3, Nk), (Nk,), device=dev, generator=g)
        k[:, :, sel == 2] = k[:, proto][:, :, sel == 2]
    elif name != "flat":
        raise ValueError(name)
    flat = lambda t: t.reshape(t.shape[0] * t.shape[1], heads * hd).bfloat16()
    return flat(q), flat(k), flat(v)


# ------------------------------------------------------------------------------------------- CPU model of the flash loop
FAULTS = ("stale_alpha", "alpha_noscale", "l_no_rescale", "mask_plus1", "drop_last_key")


def emulate_flash(q, k, v, heads, Nq, Nk, kv_div=1, fault=None):
    """The 64-key online-softmax loop of vx_flash_attn.cu in torch: keys loaded 64 rows at a time from the whole [Bkv*Nk, C]
    matrix (rows past a batch's Nk are the next batch's keys, rows past the end read as zeros) and masked from Nk on;
    fp32 m / l / O, P rounded to bf16 for O += P V, l from the unrounded P, bf16 output.  ``fault`` injects one bug:
    stale_alpha   : O is rescaled with the previous step's alpha;
    alpha_noscale : alpha = 2^(m_old - m_new) without the log2(e) / sqrt(hd) factor;
    l_no_rescale  : l is not multiplied by alpha;
    mask_plus1    : the mask starts at Nk + 1 (the first key of the next batch leaks in);
    drop_last_key : the mask starts at Nk - 1."""
    C = q.shape[1]
    hd = C // heads
    Bq, Bkv = q.shape[0] // Nq, k.shape[0] // Nk
    c = LOG2E / math.sqrt(hd)
    T = (Nk + STEP - 1) // STEP
    Q = q.float().reshape(Bq, Nq, heads, hd).transpose(1, 2)
    pad = lambda t: torch.cat([t.float(), t.new_zeros((STEP, C)).float()]).reshape(-1, heads, hd)
    K, V = pad(k), pad(v)
    kv_row0 = (torch.arange(Bq) // kv_div) * Nk
    limit = Nk + 1 if fault == "mask_plus1" else Nk - 1 if fault == "drop_last_key" else Nk
    m = torch.full((Bq, heads, Nq, 1), -math.inf)
    l = torch.zeros((Bq, heads, Nq, 1))
    O = torch.zeros((Bq, heads, Nq, hd))
    alpha_prev = torch.ones_like(l)
    for j in range(T):
        idx = kv_row0[:, None] + j * STEP + torch.arange(STEP)[None, :]
        Kj, Vj = K[idx].transpose(1, 2), V[idx].transpose(1, 2)                    # (Bq, heads, 64, hd)
        S = Q @ Kj.transpose(-1, -2)
        S[..., j * STEP + torch.arange(STEP) >= limit] = -math.inf
        m_new = torch.maximum(m, S.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new) if fault == "alpha_noscale" else torch.exp2((m - m_new) * c)
        P = torch.exp2(S * c - m_new * c)
        l = (l if fault == "l_no_rescale" else l * alpha) + P.sum(-1, keepdim=True)
        O = O * (alpha_prev if fault == "stale_alpha" else alpha) + P.bfloat16().float() @ Vj
        alpha_prev, m = alpha, m_new
    return (O / l).bfloat16().transpose(1, 2).reshape(Bq * Nq, C)


def test_bound_rejects_injected_faults():
    """The faithful model passes every family with room to spare (ratio <= 0.75), every injected fault fails the bound or
    the global criterion on at least one family, and every family catches at least one fault."""
    Bq, Nq, heads, hd = 2, 128, 2, 32
    cases = [(f, 1040) for f in FAMILIES] + [("tail", 1008)]      # Nk = 64 * 16 + 16 and 64 * 15 + 48
    caught = {f: [] for f in FAULTS}
    for fam, Nk in cases:
        g = torch.Generator().manual_seed(Nk + FAMILIES.index(fam))
        q, k, v = family_inputs(fam, g, Bq, Nq, Bq, Nk, heads, hd, n_poison=(-Nk) % STEP or 16)
        ref, ref_abs = attention_ref64(q, k, v, heads, Nq, Nk)
        worst, rel, where = bound_check(emulate_flash(q, k, v, heads, Nq, Nk), ref, ref_abs, Nk, Nq, heads)
        print(f"faithful loop  {fam:10s} Nk {Nk}: worst ratio {worst:.3f}, rel {rel:.2e}")
        assert worst <= 0.75 and rel < 4e-3, (fam, Nk, where, rel)
        for fault in FAULTS:
            worst, rel, _ = bound_check(emulate_flash(q, k, v, heads, Nq, Nk, fault=fault), ref, ref_abs, Nk, Nq, heads)
            if worst > 1 or not rel < 4e-3:
                caught[fault].append((fam, Nk, worst, rel))
    for fault, hits in caught.items():
        print(f"{fault:14s} rejected on " + ", ".join(f"{f}/{n} (ratio {w:.3g}, rel {r:.2e})" for f, n, w, r in hits))
        assert hits, f"{fault} passes every family"
    for fam, Nk in cases:
        assert any((fam, Nk) == h[:2] for hits in caught.values() for h in hits), f"{fam} / Nk {Nk} catches no fault"


# ------------------------------------------------------------------------------------------------------------ GPU cases
@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture
def serial_loop():
    """Context-free switch: serial_loop(True) routes every head dim to the serial loop until serial_loop(False)."""
    from vexpress_b200 import _ffi
    before = os.environ.get("VX_FA_V1")

    def switch(on):
        if on:
            os.environ["VX_FA_V1"] = "1"
        else:
            os.environ.pop("VX_FA_V1", None)
        _ffi.lib().vx_flash_reload_env()

    yield switch
    if before is None:
        os.environ.pop("VX_FA_V1", None)
    else:
        os.environ["VX_FA_V1"] = before
    _ffi.lib().vx_flash_reload_env()


@pytest.fixture(scope="module", autouse=True)
def _worst_ratio_summary():
    yield
    for kernel, (worst, case) in sorted(_WORST.items()):
        print(f"worst bound ratio {kernel:18s} {worst:.3f}  ({case})")


def _bordered(rows, C):
    """A NaN-filled bf16 buffer three rows taller above, five below, 8 columns wider left and 16 right (ld > C), and
    the [rows, C] slice inside it the kernel writes."""
    buf = torch.full((rows + 8, C + 24), _SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return buf, buf[3:3 + rows, 8:8 + C]


def _border_untouched(buf, rows, C):
    outside = (buf.view(torch.int16) != _SENTINEL)
    outside[3:3 + rows, 8:8 + C] = False
    n = int(outside.sum())
    return "" if n == 0 else f"{n} cells outside the output slice written, first at {outside.nonzero()[0].tolist()}"


def _judge(kernel, case, fam, out, buf, ref, ref_abs, Nk, Nq, heads):
    """Bound, global criterion, NaN inside and sentinels outside the slice -> '' or a failure message."""
    torch.cuda.synchronize()
    rows, C = out.shape
    worst, rel, where = bound_check(out, ref, ref_abs, Nk, Nq, heads)
    print(f"{kernel:18s} {case} {fam:10s}: worst ratio {worst:.3f}, rel {rel:.2e}")
    if worst > _WORST.get(kernel, (-1.0, ""))[0]:
        _WORST[kernel] = (worst, f"{case} {fam}")
    bad = []
    if not worst <= 1:
        bad.append(f"bound exceeded, {where}")
    if not rel < 4e-3:
        bad.append(f"global rel {rel:.3e}")
    if torch.isnan(out.float()).any():
        bad.append("NaN left in the output")
    border = _border_untouched(buf, rows, C)
    if border:
        bad.append(border)
    return f"{kernel} {case} {fam}: " + "; ".join(bad) if bad else ""


def _flash_kernel(Nk, hd, serial):
    if Nk < 16 or Nk % 16:
        return "generic"
    return "serial" if serial or hd > 56 else "pipelined"


def _run_flash(ops, families, Bq, Nq, Nk, heads, hd, kv_div=1, serial=False, kv=None):
    """flash_attention over each family with K / V as the column halves of one [rows, 2C] tensor and out as an interior
    slice of a NaN-bordered buffer.  ``kv`` overrides the inputs (a fixed call pattern) and runs them as family 'given'."""
    Bkv = (Bq + kv_div - 1) // kv_div
    C = heads * hd
    kernel = _flash_kernel(Nk, hd, serial)
    case = f"Bq {Bq} Nq {Nq} Nk {Nk} {heads}x{hd} kv_div {kv_div}"
    fails = []
    for fam in families:
        if kv is None:
            g = torch.Generator(device="cuda").manual_seed(Bq * Nq + Nk + hd + FAMILIES.index(fam))
            q, k, v = family_inputs(fam, g, Bq, Nq, Bkv, Nk, heads, hd, n_poison=min(Nk, (-Nk) % STEP or 16))
            kvt = torch.cat([k, v], 1)
        else:
            q, kvt = kv
            fam = "given"
        k, v = kvt[:, :C], kvt[:, C:]
        buf, out = _bordered(Bq * Nq, C)
        ops.flash_attention(q, k, v, heads, Nq, Nk, kv_div, out=out)
        ref, ref_abs = attention_ref64(q, k, v, heads, Nq, Nk, kv_div)
        fails.append(_judge(kernel, case, fam, out, buf, ref, ref_abs, Nk, Nq, heads))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


ALL = FAMILIES
SHORT = ("flat", "peaked", "poison", "degenerate")


# pipelined loop (hd <= 56): (Bq, Nq, Nk) = two consumer warpgroups with a ragged last tile and a masked tail (Nk 64 * 16
# + 16), one warpgroup with a 48-key tail, fewer steps than ring stages (T = 3), a single step (T = 1)
@pytest.mark.gpu
@pytest.mark.parametrize("Bq,Nq,Nk", [(2, 200, 1040), (2, 64, 1072), (2, 64, 192), (3, 200, 64)])
@pytest.mark.parametrize("hd", [8, 16, 24, 32, 40, 48, 56])
def test_pipelined_flash_within_bound(ops, hd, Bq, Nq, Nk):
    _run_flash(ops, ALL, Bq, Nq, Nk, 3, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("Bq,kv_div", [(2, 1), (16, 16)])
def test_pipelined_flash_production_within_bound(ops, Bq, kv_div):
    """The 64 x 64-latent self-attention and the reference attention of a 16-frame window (one bank, kv_div = f)."""
    _run_flash(ops, ("flat", "peaked", "rising", "poison"), Bq, 4096, 4096, 8, 40, kv_div)


# serial loop (hd > 56), including the padded widths 72 / 120 / 200 (Q / K / V tiles zero-padded to 80 / 128 / 208)
@pytest.mark.gpu
@pytest.mark.parametrize("hd", [64, 72, 80, 96, 120, 128, 160, 200, 256])
def test_serial_flash_within_bound(ops, hd):
    _run_flash(ops, ALL, 2, 200, 1040, 2, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("Bq,Nq,hd", [(2, 1024, 80), (2, 256, 160), (4, 144, 160)])
def test_serial_flash_production_within_bound(ops, Bq, Nq, hd):
    _run_flash(ops, ("flat", "peaked", "rising", "poison"), Bq, Nq, Nq, 8, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("hd,serial", [(40, False), (40, True), (80, False)])
def test_flash_ragged_kv_div_within_bound(ops, serial_loop, hd, serial):
    """Bq = 5 query batches over Bkv = 3 kv batches (kv_div = 2): the last kv batch serves one query batch."""
    serial_loop(serial)
    _run_flash(ops, ("flat", "peaked", "tail", "poison"), 5, 200, 1040, 4, hd, kv_div=2, serial=serial)


@pytest.mark.gpu
@pytest.mark.parametrize("Nq", [5, 33])
@pytest.mark.parametrize("hd", [8, 64, 160])
@pytest.mark.parametrize("Nk", [1, 4, 15, 36, 1000, 3000])
def test_generic_attention_within_bound(ops, Nk, hd, Nq):
    """Key counts the tensor-core tiling cannot express (Nk < 16 or Nk % 16 != 0), up to the kernel's limit of 3072."""
    _run_flash(ops, SHORT + (("tail",) if Nk > 4 else ()), 2, Nq, Nk, 3, hd)


@pytest.mark.gpu
def test_generic_attention_prologue_call_within_bound(ops):
    """The prologue's cross-attention exactly: 12 heads x hd 64, 5 latent queries over 15 keys, K / V the column halves of
    one to_kv output [rows, 2 * 768]."""
    g = torch.Generator(device="cuda").manual_seed(215)
    q = torch.randn(2 * 5, 768, device="cuda", generator=g).bfloat16()
    kv = (2 * torch.randn(2 * 15, 2 * 768, device="cuda", generator=g)).bfloat16()
    _run_flash(ops, ("given",), 2, 5, 15, 12, 64, kv=(q, kv))


def _run_temporal(ops, families, b, f, HW, heads, hd):
    """temporal_attention over each family.  Inputs are generated as (b HW) batches of f tokens, the layout of the
    reference, and moved to the kernel's (b f HW) rows; poison goes to the first frames of b >= 1, which a kernel reading
    past its own f frames at one pixel would reach."""
    C = heads * hd
    kernel = "temporal mma" if f <= 16 else "temporal cuda-core"
    fpad = 16 if f <= 16 else 32
    case = f"b {b} f {f} HW {HW} {heads}x{hd}"
    to_kernel = lambda t: t.reshape(b, HW, f, C).transpose(1, 2).reshape(b * f * HW, C)
    fails = []
    for fam in families:
        g = torch.Generator(device="cuda").manual_seed(b * 1000 + f * 31 + hd + FAMILIES.index(fam))
        q, k, v = family_inputs(fam, g, b * HW, f, b * HW, f, heads, hd, poison_from=HW, n_poison=min(f, fpad - f) or 1)
        qkv = torch.cat([to_kernel(q), to_kernel(k), to_kernel(v)], 1)
        buf, out = _bordered(b * f * HW, C)
        ops.temporal_attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], b, f, HW, heads, out=out)
        ref, ref_abs = attention_ref64(q, k, v, heads, f, f)
        torch.cuda.synchronize()
        out_ref_layout = out.reshape(b, f, HW, C).transpose(1, 2).reshape(b * HW * f, C)
        fails.append(_judge(kernel, case, fam, out_ref_layout, buf, ref, ref_abs, f, f, heads))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("b,HW", [(1, 8), (2, 3)])
@pytest.mark.parametrize("hd", [8, 16, 32, 40, 80, 160])
@pytest.mark.parametrize("f", [1, 2, 7, 8, 9, 15, 16, 17, 20, 24, 31, 32])
def test_temporal_attention_within_bound(ops, f, hd, b, HW):
    """f <= 16: the mma kernel (16 x 16 fragments, frames >= f masked); f > 16: the CUDA-core kernel (fpad 32; hd 160
    stages K / V as bf16)."""
    _run_temporal(ops, SHORT, b, f, HW, 3, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("HW,hd", [(4096, 40), (1024, 80), (256, 160)])
def test_temporal_attention_production_window_within_bound(ops, HW, hd):
    """The default 24-frame context window at each UNet level."""
    _run_temporal(ops, ("flat", "peaked", "poison"), 2, 24, HW, 8, hd)


def _run_smallkv(ops, families, frames, rpf, heads, hd, Lk):
    C = heads * hd
    kernel = "smallkv mma" if rpf % 16 == 0 and hd in (8, 40, 80, 160) else "smallkv cuda-core"
    case = f"frames {frames} rows/frame {rpf} {heads}x{hd} Lk {Lk}"
    fails = []
    for fam in families:
        g = torch.Generator(device="cuda").manual_seed(frames * rpf + hd + Lk + FAMILIES.index(fam))
        q, k, v = family_inputs(fam, g, frames, rpf, frames, Lk, heads, hd, n_poison=min(Lk, 8 - Lk) or 1)
        kv = torch.cat([k, v], 1)
        buf, out = _bordered(frames * rpf, C)
        ops.smallkv_attention(q, kv[:, :C], kv[:, C:], rpf, heads, Lk, out=out)
        ref, ref_abs = attention_ref64(q, k, v, heads, rpf, Lk)
        fails.append(_judge(kernel, case, fam, out, buf, ref, ref_abs, Lk, rpf, heads))
    fails = [f for f in fails if f]
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("Lk", [1, 2, 5, 8])
@pytest.mark.parametrize("hd", [8, 40, 80, 160])
def test_smallkv_mma_within_bound(ops, hd, Lk):
    _run_smallkv(ops, SHORT, 3, 48, 3, hd, Lk)


@pytest.mark.gpu
@pytest.mark.parametrize("Lk", [1, 5, 8])
@pytest.mark.parametrize("hd", [24, 64])
@pytest.mark.parametrize("rpf", [20, 4])
def test_smallkv_cuda_core_within_bound(ops, rpf, hd, Lk):
    """rows_per_frame % 16 != 0 (or a head dim without an mma instantiation): one thread per (row, head)."""
    _run_smallkv(ops, SHORT, 3, rpf, 3, hd, Lk)


@pytest.mark.gpu
def test_smallkv_production_within_bound(ops):
    """Audio cross-attention at the 64 x 64 level: 2 x 16 frames x 4096 rows, 8 x 40, 5 audio tokens per frame."""
    _run_smallkv(ops, ("flat", "peaked", "poison"), 32, 4096, 8, 40, 5)
