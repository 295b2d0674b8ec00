"""Ping-pong at the 128- and 160-column tiles, and on every convolution producer, against the cooperative schedule, bit
for bit.

As in test_gemm_pingpong_gpu.py, every case runs one call under VX_GEMM_PP=0 (cooperative) and VX_GEMM_PP=1
(ping-pong) and compares the raw bits of the whole output buffer; operands, residuals and outputs sit inside NaN borders.
The launch log (VX_GEMM_VERBOSE) confirms the schedule, the width and, for the stride-1 convolutions, the producer (row
reuse or tap by tap) each arm ran."""
import os
import re
import sys
import tempfile

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gemm_pingpong_gpu import NAN16, _bordered, _check, _gemm_case, _geglu_inputs, _in_nan, gemm_env, ops  # noqa: E402,F401

WIDE = [128, 160]


def _logged(fn):
    """Run fn with the C library's stderr captured: (result, [(bn, pp, rr) of every GEMM launch])."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            r = fn()
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        log = f.read().decode()
    return r, [tuple(int(v) for v in m) for m in re.findall(r"bn=(\d+) pp=(\d+) rr=(\d+)", log)]


def _both(gemm_env, run, bn=None, rr=None):
    """run() under both schedules -> [coop buffer, pp buffer]; asserts schedule, width and producer from the log"""
    bufs = []
    for pp in (0, 1):
        gemm_env(VX_GEMM_PP=pp, VX_GEMM_VERBOSE=1)
        buf, launches = _logged(run)
        assert launches and all(p == pp and (bn is None or b == bn) and (rr is None or r == rr)
                                for b, p, r in launches), (pp, launches)
        bufs.append(buf)
    return bufs


# ---------------------------------------------------------------- plain GEMM
@pytest.mark.gpu
@pytest.mark.parametrize("block_n", WIDE)
@pytest.mark.parametrize("bias,div,scale,residual", [
    (False, 0, 1.0, False), (True, 0, 1.0, False), (True, 7, 1.0, False), (True, 129, 0.37, False),
    (True, 0, -1.5, True), (False, 300, 0.37, True)])
def test_wide_linear_epilogues(ops, gemm_env, block_n, bias, div, scale, residual):
    """N = 3840 divides by 128 and 160."""
    _gemm_case(ops, gemm_env, 300, 200, 3840, bias=bias, div=div, scale=scale, residual=residual, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", WIDE)
@pytest.mark.parametrize("M,K", [(1, 320), (129, 72), (128 * 133 + 1, 448)])
def test_wide_rows_and_k_tails(ops, gemm_env, block_n, M, K):
    _gemm_case(ops, gemm_env, M, K, 640, div=7, scale=-1.5, residual=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", WIDE)
@pytest.mark.parametrize("K1,K2", [(64, 8), (320, 72), (320, 320)])
def test_wide_split_k(ops, gemm_env, block_n, K1, K2):
    _gemm_case(ops, gemm_env, 300, K1, 640, K2=K2, residual=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", WIDE)
def test_wide_fp32_out(ops, gemm_env, block_n):
    _gemm_case(ops, gemm_env, 300, 200, 640, div=7, scale=0.125, out_f32=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", WIDE)
@pytest.mark.parametrize("case", ["odd items per CTA", "fewer tiles than SMs", "one tile"])
def test_wide_item_counts(ops, gemm_env, block_n, case):
    """Odd: three tiles per CTA (warpgroup 0 takes two, warpgroup 1 one).  Fewer tiles than SMs: one tile per CTA, so
    warpgroup 1 has none.  One tile: a single CTA."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M, N = {"odd items per CTA": (128 * 3 * sms, block_n), "fewer tiles than SMs": (128 * 5 - 3, 2 * block_n),
            "one tile": (100, block_n)}[case]
    _gemm_case(ops, gemm_env, M, 320, N, residual=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(300, 320, 512), (129, 640, 2560), (1000, 1280, 256), (128 * 133 + 1, 320, 2560)])
def test_geglu_128_packing(ops, gemm_env, M, K, N):
    """GEGLU packed per 128-column tile (ping-pong) against the default 256-column packing (cooperative), per output
    column; and both schedules on the 128-column packing."""
    a, w, b = _geglu_inputs(M, K, N, M + K)
    a = _in_nan(a)
    outs = {}
    for pp, bn in ((0, 256), (0, 128), (1, 128)):
        wp, bp, _ = ops.pack_geglu(w, b, bn)
        wp = _in_nan(wp)

        def run():
            buf, out = _bordered(M, N // 2)
            ops.gemm(a, wp, bp, geglu=True, block_n=bn, out=out)
            return buf
        gemm_env(VX_GEMM_PP=pp, VX_GEMM_VERBOSE=1)
        buf, launches = _logged(run)
        assert [l[:2] for l in launches] == [(bn, pp)], launches
        outs[(pp, bn)] = buf
    _check([outs[(0, 256)], outs[(1, 128)]])
    _check([outs[(0, 128)], outs[(1, 128)]])


# ---------------------------------------------------------------- convolutions
def _conv_run(ops, kind, NB, H, W, C, Cout, block_n, seed, epilogue=True):
    """run() of one conv3x3 (s1, with bias, per-frame bias2, scale and residual), conv3x3_s2 or upconv3x3 call; the input is
    frames 1..NB of a buffer whose frames 0 and NB + 1 are NaN, the output sits inside a NaN border.  The weights are
    contiguous: the conv entry points take no weight stride."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    taps = 4 if kind == "ups" else 9
    xb = torch.full((NB + 2, H, W, C), NAN16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    xb[1:NB + 1] = rnd(NB, H, W, C).bfloat16()
    x = xb[1:NB + 1]
    w = (rnd(Cout * (4 if kind == "ups" else 1), taps * C) / (taps * C) ** 0.5).bfloat16()
    b = rnd(Cout)
    Ho, Wo = (H // 2, W // 2) if kind.startswith("s2") else (H, W)
    rows = NB * Ho * Wo * (4 if kind == "ups" else 1)
    b2 = rnd(NB, Cout) if epilogue else None
    r = _in_nan(rnd(rows, Cout).bfloat16()) if epilogue else None

    def run():
        buf, out = _bordered(rows, Cout)
        if kind == "s1":
            ops.conv3x3(x, w, b, bias2=b2, bias2_div=H * W, scale=0.37 if epilogue else 1.0, residual=r, out=out,
                        block_n=block_n)
        elif kind == "s2":
            ops.conv3x3_s2(x, w, b, pad_lo=1, out=out, block_n=block_n)
        elif kind == "s2p0":
            ops.conv3x3_s2(x, w, b, pad_lo=0, out=out, block_n=block_n)
        else:
            ops.upconv3x3(x, w, b, out=out, block_n=block_n)
        return buf
    return run


# (kind, NB, H, W, C, Cout, block_n, producer): row reuse where three stages fit beside two staging tiles (rr = 1), tap by
# tap elsewhere; row tails (tiles of 96 rows), tile counts below the SM count and odd per CTA
CONV_CASES = [
    ("s1", 4, 32, 32, 128, 640, 64, 1),      # row reuse, 4 image rows per tile
    ("s1", 4, 16, 16, 128, 256, 64, 1),      # row reuse, 8 image rows per tile
    ("s1", 4, 16, 16, 128, 192, 96, 1),      # row reuse at the widest width it fits beside two staging tiles
    ("s1", 6, 64, 64, 64, 320, 64, 1),       # row reuse, 2 image rows per tile (the 64 x 64 level's ping-pong width)
    ("s1", 2, 64, 64, 64, 320, 160, 0),      # forced tap by tap (VX_CONV_RR=0 below) at 160
    ("s1", 3, 48, 48, 64, 320, 160, 0),      # 96-row tiles (2 image rows of 48): tap by tap
    ("s1", 2, 96, 96, 64, 256, 128, 0),      # 96-pixel-wide rows: 96-row tiles
    ("s1", 6, 8, 8, 128, 320, 160, 0),       # 2 frames per tile; 3 row tiles, fewer tiles than SMs
    ("s1", 2, 8, 8, 64, 160, 160, 0),        # one tile
    ("s2", 4, 64, 64, 64, 320, 160, None),   # stride 2, pad 1
    ("s2p0", 2, 32, 32, 64, 256, 128, None),  # stride 2, pad (0, 1, 0, 1)
    ("ups", 4, 16, 16, 64, 320, 160, None),  # folded nearest-2x upsample
    ("ups", 2, 48, 48, 64, 256, 128, None),  # upsample with 96-row tiles of 48-wide rows
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,NB,H,W,C,Cout,block_n,rr", CONV_CASES)
def test_conv_producers(ops, gemm_env, kind, NB, H, W, C, Cout, block_n, rr):
    run = _conv_run(ops, kind, NB, H, W, C, Cout, block_n, NB * 131 + H * 7 + Cout + block_n)
    if (kind, H, block_n) == ("s1", 64, 160):
        os.environ["VX_CONV_RR"] = "0"
    try:
        bufs = _both(gemm_env, run, bn=block_n, rr=rr)
    finally:
        os.environ.pop("VX_CONV_RR", None)
        from vexpress_b200 import _ffi
        _ffi.lib().vx_gemm_reload_env()
    _check(bufs)


@pytest.mark.gpu
def test_conv_odd_items_per_cta(ops, gemm_env):
    """Three 128 x 160 tiles per CTA (tap by tap: 2 frames of 8 x 8 per tile), so warpgroup 0 takes two and warpgroup 1 one."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    run = _conv_run(ops, "s1", 2 * 3 * sms, 8, 8, 64, 160, 160, 17)
    _check(_both(gemm_env, run, bn=160, rr=0))


def _conv_forward_shapes():
    """(kind, NB, H, W, C, Cout) of every convolution of one benchmark UNet forward (32 frames), from tools/gemm_ab.py."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("gemm_ab", os.path.join(os.path.dirname(os.path.dirname(
        os.path.abspath(__file__))), "tools", "gemm_ab.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = []
    for (kind, M, N, K), _ in mod.unique_shapes():
        side = int(round((M / 32) ** 0.5))
        if kind == "upconv3x3":
            out.append(("ups", 32, side // 2, side // 2, K // 4, N))
        elif kind == "conv3x3 s2":
            out.append(("s2", 32, 2 * side, 2 * side, K // 9, N))
        elif kind == "conv3x3":
            out.append(("s1", 32, side, side, K // 9, N))
    return out


@pytest.mark.gpu
def test_conv_production_shapes(ops, gemm_env):
    """Every convolution of one benchmark UNet forward at its production shape: the default rule's choice and both forced
    schedules agree bit for bit, and the default launch uses the producer the cooperative one uses."""
    for kind, NB, H, W, C, Cout in _conv_forward_shapes():
        run = _conv_run(ops, kind, NB, H, W, C, Cout, 0, H + C + Cout, epilogue=kind == "s1")
        outs, logs = [], []
        for pp in (0, 1, None):
            if pp is None:
                gemm_env(VX_GEMM_VERBOSE=1)
            else:
                gemm_env(VX_GEMM_PP=pp, VX_GEMM_VERBOSE=1)
            buf, launches = _logged(run)
            outs.append(buf)
            logs.append(launches)
        _check([outs[0], outs[1]])
        _check([outs[0], outs[2]])
        assert logs[0][0][2] == logs[2][0][2], (kind, NB, H, W, C, Cout, logs)   # the same producer
        del outs
