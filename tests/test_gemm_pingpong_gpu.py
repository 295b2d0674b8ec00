"""Ping-pong GEMM schedule against the cooperative one, bit for bit.

Both schedules of gemm_wgmma_kernel add the same products in the same K order and round at the same points; only which
warpgroup computes a tile, and when, differs.  So every case runs one ops.gemm call twice, with VX_GEMM_PP=0 (cooperative)
and VX_GEMM_PP=1 (ping-pong), and compares the raw bits of the whole output buffer: the output slice sits inside a NaN
border with ld > N that must survive, and the operands and residuals are interior views of NaN buffers.  The launch log
(VX_GEMM_VERBOSE) confirms that each arm ran the schedule it asked for."""
import importlib.util
import os
import re
import sys
import tempfile

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAN16, NAN32 = 0x7FC0, 0x7FC00000


@pytest.fixture(scope="module")
def ops():
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    return ops


@pytest.fixture
def gemm_env():
    """gemm_env(VX_GEMM_PP=.., ...) sets exactly these switches and makes the library re-read them; restored at the end."""
    from vexpress_b200 import _ffi
    names = ("VX_GEMM_PP", "VX_GEMM_STAGES", "VX_GEMM_NBUF", "VX_GEMM_VERBOSE")
    before = {n: os.environ.get(n) for n in names}

    def restore():
        for n, v in before.items():
            if v is None:
                os.environ.pop(n, None)
            else:
                os.environ[n] = v

    def switch(**kv):
        restore()
        for n, v in kv.items():
            os.environ[n] = str(v)
        _ffi.lib().vx_gemm_reload_env()

    yield switch
    restore()
    _ffi.lib().vx_gemm_reload_env()


def _nan_buf(rows, cols, dtype):
    bits = torch.full((rows + 8, cols + 24), NAN32 if dtype == torch.float32 else NAN16,
                      dtype=torch.int32 if dtype == torch.float32 else torch.int16, device="cuda")
    return bits.view(dtype)


def _bordered(rows, cols, dtype=torch.bfloat16):
    """NaN buffer three rows taller above, five below, 8 columns wider left and 16 right; the [rows, cols] view inside."""
    buf = _nan_buf(rows, cols, dtype)
    return buf, buf[3:3 + rows, 8:8 + cols]


def _in_nan(t):
    if t is None:
        return None
    _, view = _bordered(*t.shape, t.dtype)
    view.copy_(t)
    return view


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _logged(fn):
    """Run fn with the C library's stderr captured: (result, [(bn, pp) of every GEMM launch])."""
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
    return r, [(int(b), int(p)) for b, p in re.findall(r"bn=(\d+) pp=(\d+)", log)]


def _both(gemm_env, run, extra=None, expect_pp=True):
    """run(out_view) under the cooperative and the ping-pong schedule -> (coop buffer, pp buffer); asserts the launch log"""
    bufs = []
    for pp in (0, 1):
        gemm_env(VX_GEMM_PP=pp, VX_GEMM_VERBOSE=1, **(extra or {}))
        buf, launches = _logged(run)
        assert launches and all(p == (pp if expect_pp else 0) for _, p in launches), (pp, launches)
        bufs.append(buf)
    return bufs


def _check(bufs, nan_inside_ok=False):
    coop, pp = bufs
    assert torch.equal(_bits(coop), _bits(pp)), \
        f"ping-pong differs from cooperative at {(_bits(coop) != _bits(pp)).nonzero()[:4].tolist()}"
    inner = coop[3:-5, 8:-16]
    border = _bits(coop).clone()
    border[3:-5, 8:-16] = NAN32 if coop.dtype == torch.float32 else NAN16
    assert bool((border == (NAN32 if coop.dtype == torch.float32 else NAN16)).all()), "the NaN border was written"
    if not nan_inside_ok:
        assert not torch.isnan(inner.float()).any(), "NaN left inside the output"


def _gemm_case(ops, gemm_env, M, K1, N, *, K2=0, bias=True, div=0, scale=1.0, residual=False, out_f32=False, block_n=0,
               seed=0, extra=None):
    g = torch.Generator(device="cuda").manual_seed(seed + 7919 * M + 31 * N + K1 + 3 * K2)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    a = _in_nan(rnd(M, K1).bfloat16())
    a2 = _in_nan(rnd(M, K2).bfloat16()) if K2 else None
    w = _in_nan((rnd(N, K1 + K2) / (K1 + K2) ** 0.5).bfloat16())
    b = rnd(N) if bias else None
    b2 = rnd((M - 1) // div + 1, N) if div else None
    r = _in_nan(rnd(M, N).bfloat16()) if residual else None
    dtype = torch.float32 if out_f32 else torch.bfloat16

    def run():
        buf, out = _bordered(M, N, dtype)
        ops.gemm(a, w, b, a2=a2, bias2=b2, bias2_div=div or 1, scale=scale, residual=r, out=out, block_n=block_n,
                 out_f32=out_f32)
        return buf
    _check(_both(gemm_env, run, extra))


@pytest.mark.gpu
@pytest.mark.parametrize("M,K", [(1, 320), (127, 320), (129, 72), (300, 8), (300, 200), (300, 1280), (128 * 133 + 1, 448)])
def test_rows_and_k_tails(ops, gemm_env, M, K):
    _gemm_case(ops, gemm_env, M, K, 256, div=7, scale=-1.5, residual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [32, 64, 96])
@pytest.mark.parametrize("bias,div,scale,residual", [
    (False, 0, 1.0, False), (True, 0, 1.0, False), (True, 7, 1.0, False), (True, 129, 0.37, False),
    (True, 0, -1.5, True), (False, 300, 0.37, True)])
def test_every_linear_epilogue_and_block_n(ops, gemm_env, block_n, bias, div, scale, residual):
    """N = 3840 divides by every ping-pong column-tile width."""
    _gemm_case(ops, gemm_env, 300, 200, 3840, bias=bias, div=div, scale=scale, residual=residual, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("K2", [8, 72, 320])
@pytest.mark.parametrize("K1", [64, 320])
def test_split_k(ops, gemm_env, K1, K2):
    _gemm_case(ops, gemm_env, 300, K1, 640, K2=K2, residual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("N,block_n", [(64, 0), (96, 0), (320, 0), (3840, 96)])
def test_fp32_out(ops, gemm_env, N, block_n):
    _gemm_case(ops, gemm_env, 300, 200, N, div=7, scale=0.125, out_f32=True, block_n=block_n)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["odd items per CTA", "fewer tiles than SMs", "one tile"])
def test_item_counts(ops, gemm_env, case):
    """Odd: three 128 x 96 tiles per CTA, so warpgroup 0 takes two and warpgroup 1 one.  Fewer tiles than SMs: every
    CTA has one tile and warpgroup 1 none.  One tile: a single CTA."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M, N = {"odd items per CTA": (128 * 3 * sms, 96), "fewer tiles than SMs": (128 * 5 - 3, 192),
            "one tile": (100, 96)}[case]
    _gemm_case(ops, gemm_env, M, 320, N, residual=True, block_n=96)


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value", [("VX_GEMM_STAGES", 2), ("VX_GEMM_STAGES", 3), ("VX_GEMM_STAGES", 7)])
def test_stages_bit_identical(ops, gemm_env, knob, value):
    """Ring depth changes nothing in the arithmetic of either schedule: forced depth against the default depth, both
    schedules (more tiles than SMs, K = 7 blocks)."""
    _gemm_case(ops, gemm_env, 128 * 133 + 1, 448, 320, div=7, residual=True, block_n=64)
    _gemm_case(ops, gemm_env, 128 * 133 + 1, 448, 320, div=7, residual=True, block_n=64, extra={knob: value})
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(128 * 133 + 1, 448, device="cuda", generator=g).bfloat16()
    w = (torch.randn(320, 448, device="cuda", generator=g) / 21).bfloat16()
    outs = []
    for extra in ({}, {knob: value}):
        gemm_env(VX_GEMM_PP=1, **extra)
        outs.append(ops.gemm(a, w, block_n=64))
    assert torch.equal(outs[0], outs[1])


def _geglu_inputs(M, K, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    return a, w, b


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(300, 320, 512), (129, 640, 2560), (1000, 1280, 256)])
def test_geglu_both_packings(ops, gemm_env, M, K, N):
    """GEGLU packed per 64-column tile (ping-pong) against the 256-column packing (cooperative), per output column;
    and both schedules on the 64-column packing."""
    a, w, b = _geglu_inputs(M, K, N, M + K)
    a = _in_nan(a)
    outs = {}
    for pp, bn in ((0, 256), (0, 64), (1, 64)):
        wp, bp, _ = ops.pack_geglu(w, b, bn)
        wp = _in_nan(wp)

        def run():
            buf, out = _bordered(M, N // 2)
            ops.gemm(a, wp, bp, geglu=True, block_n=bn, out=out)
            return buf
        gemm_env(VX_GEMM_PP=pp, VX_GEMM_VERBOSE=1)
        buf, launches = _logged(run)
        assert launches == [(bn, pp)], launches
        outs[(pp, bn)] = buf
    _check([outs[(0, 256)], outs[(1, 64)]])
    _check([outs[(0, 64)], outs[(1, 64)]])


def _forward_shapes():
    spec = importlib.util.spec_from_file_location("gemm_ab", os.path.join(ROOT, "tools", "gemm_ab.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return [s for (s, _) in mod.unique_shapes() if not s[0].startswith(("conv", "upconv"))], mod.RESIDUAL


@pytest.mark.gpu
def test_production_shapes(ops, gemm_env):
    """Every plain-GEMM shape of one benchmark UNet forward (b = 2, f = 16, 64x64), with the epilogue it has there: the
    default rule's choice and both forced schedules agree bit for bit."""
    shapes, residual_kinds = _forward_shapes()
    bad = []
    for kind, M, N, K in shapes:
        a, w, b = _geglu_inputs(M, K, N, M + N + K)
        geglu = "geglu" in kind
        if geglu:
            w, b, _ = ops.pack_geglu(w, b, 64)
        r = torch.randn(M, N, device="cuda").bfloat16() if kind in residual_kinds else None
        outs = []
        for pp in (0, 1, None):
            if pp is None:
                gemm_env()
            else:
                gemm_env(VX_GEMM_PP=pp)
            outs.append(ops.gemm(a, w, b, geglu=True, block_n=64) if geglu else ops.gemm(a, w, b, residual=r))
        if not (torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])):
            bad.append((kind, M, N, K))
        del a, w, r, outs
    assert not bad, bad
