"""A/B timing of the GEMM consumer schedules (cooperative, ping-pong at each width) on the GEMM / convolution shapes of
one UNet forward of the benchmark workload (b = 2 CFG halves x f = 16 frames, 64x64 latents: 32 frames per launch).

    python tools/gemm_ab.py [--min-ms 300] [--rounds 3] [--widths 64,96,128,160] [--baseline-lib LIB] [--plan] [--json FILE]

The shape list restates the launches `UNetEngine.forward_frames` issues (4 down levels of 320 / 640 / 1280 / 1280 channels,
the mid block, 4 up levels with 3 resnets each; spatial transformers at the 64 / 32 / 16 levels, motion modules
everywhere).  Per shape these arms alternate, arm by arm, `--rounds` times:
  parent  (with --baseline-lib: a libvxb200.so built from an earlier commit) that library's default choice;
  coop    cooperative schedule (VX_GEMM_PP=0) at the column tile the cost model picks for it;
  pp<bn>  ping-pong schedule (VX_GEMM_PP=1) at column tile bn, for every width in --widths that divides N (GEGLU: and is a
          multiple of 64); a stride-1 convolution uses row reuse where two ring stages fit beside two staging tiles;
  default the library's default rule (timed only when it differs from every arm above).
GEGLU weights are packed for each arm's tile; the parent, coop and default arms use the 256-column packing.
One sample is as many back-to-back launches as fill at least `--min-ms` between two CUDA events; the SM clock is read by a
thread while that window runs.  Prints ms per launch (median over rounds, with the spread), TFLOP/s (2 M N K), the
L2 -> shared-memory operand bytes per FLOP of the tile ((128 + bn) / (128 bn): every K block moves a 128-row A box and a
bn-row W box), whether every arm's output is bit-identical to coop's, and per forward the sum over launches for the
parent, coop, the default rule and the fastest arm of every shape.  The card name, power limit and the median sampled SM
clock are printed with the table.  Inputs come from a seed.
`--plan` prints the shape / FLOP table and stops; timing without a CUDA device is an error."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 32
RESIDUAL = ("attn out", "ff2", "proj_out")   # GEMMs whose epilogue adds the residual stream


def forward_launches():
    """(kind, M, N, K) of every GEMM / conv launch of one forward; conv K = taps x Cin."""
    ops = []
    g = lambda kind, M, N, K: ops.append((kind, M, N, K))

    def spatial(C, M):
        g("proj_in", M, C, C); g("qkv", M, 3 * C, C); g("attn out", M, C, C)
        g("q (attn1_5)", M, C, C); g("attn out", M, C, C); g("q (attn2)", M, C, C); g("attn out", M, C, C)
        g("ff1 geglu", M, 8 * C, C); g("ff2", M, C, 4 * C); g("proj_out", M, C, C)

    def motion(C, M):
        g("proj_in", M, C, C)
        for _ in range(2):
            g("qkv", M, 3 * C, C); g("attn out", M, C, C)
        g("ff1 geglu", M, 8 * C, C); g("ff2", M, C, 4 * C); g("proj_out", M, C, C)

    def resnet(Cin, Cout, M):
        g("conv3x3", M, Cout, 9 * Cin); g("conv3x3", M, Cout, 9 * Cout)
        if Cin != Cout:
            g("shortcut", M, Cout, Cin)

    side, ch = [64, 32, 16, 8], [320, 640, 1280, 1280]
    cin, skips = 320, [320]
    for i in range(4):
        M, C = FRAMES * side[i] ** 2, ch[i]
        for _ in range(2):
            resnet(cin, C, M); cin = C
            if i < 3:
                spatial(C, M)
            motion(C, M); skips.append(C)
        if i < 3:
            g("conv3x3 s2", FRAMES * side[i + 1] ** 2, C, 9 * C); skips.append(C)
    M = FRAMES * 64
    resnet(1280, 1280, M); spatial(1280, M); motion(1280, M); resnet(1280, 1280, M)
    cin = 1280
    for i, (s, C) in enumerate(zip([8, 16, 32, 64], [1280, 1280, 640, 320])):
        M = FRAMES * s * s
        for _ in range(3):
            resnet(cin + skips.pop(), C, M); cin = C
            if i > 0:
                spatial(C, M)
            motion(C, M)
        if i < 3:
            g("upconv3x3", FRAMES * (2 * s) ** 2, C, 4 * C)   # folded nearest-2x upsample: 4 taps per output parity
    return ops


def unique_shapes():
    count, order = {}, []
    for kind, M, N, K in forward_launches():
        key = (kind, M, N, K)
        if key not in count:
            order.append(key)
        count[key] = count.get(key, 0) + 1
    return [(k, count[k]) for k in order]


def smi(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else "unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-ms", type=float, default=300.0, help="least length of one timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plan", action="store_true")
    ap.add_argument("--json", default=None, help="also write the table to this file")
    ap.add_argument("--widths", default="64,96,128,160", help="ping-pong column tiles to time")
    ap.add_argument("--baseline-lib", default=None, help="libvxb200.so of an earlier build, timed as the parent arm")
    args = ap.parse_args()

    shapes = unique_shapes()
    total = sum(2.0 * M * N * K * c for (_, M, N, K), c in shapes)
    print(f"{'kind':12s} {'M':>7s} {'N':>6s} {'K':>6s} {'launches':>8s} {'TFLOP':>7s}")
    for (kind, M, N, K), c in shapes:
        print(f"{kind:12s} {M:7d} {N:6d} {K:6d} {c:8d} {2.0 * M * N * K * c / 1e12:7.3f}")
    print(f"total: {sum(c for _, c in shapes)} launches, {total / 1e12:.2f} TFLOP per forward")
    if args.plan:
        return

    import torch
    if not torch.cuda.is_available():
        sys.exit("gemm_ab: no CUDA device; timings are only taken on the GPU")
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    device = smi("name,power.limit,clocks.max.sm")
    print("device:", device)
    lib = _ffi.lib()

    def set_env(**kv):
        for k, v in kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        _ffi.lib().vx_gemm_reload_env()   # the library the next arm runs on

    def launch_info(run):
        """(bn, pp, rr) of one launch, from the VX_GEMM_VERBOSE log on fd 2 (rr: None where the log does not say)"""
        set_env(VX_GEMM_VERBOSE=1)
        sys.stderr.flush()
        saved = os.dup(2)
        with tempfile.TemporaryFile() as f:
            os.dup2(f.fileno(), 2)
            try:
                run()
                torch.cuda.synchronize()
            finally:
                os.dup2(saved, 2)
                os.close(saved)
            f.seek(0)
            log = f.read().decode()
        set_env(VX_GEMM_VERBOSE=None)
        m = re.findall(r"bn=(\d+) pp=(\d+)(?: rr=(\d+))?", log)
        return (int(m[-1][0]), int(m[-1][1]), int(m[-1][2]) if m[-1][2] else None) if m else (0, 0, None)

    def window(run, n, sample):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        clk = []
        e0.record()
        th = threading.Thread(target=lambda: clk.append(smi("clocks.sm")))   # runs while the launches execute
        if sample:
            th.start()
        for _ in range(n):
            run()
        e1.record()
        e1.synchronize()
        if sample:
            th.join()
        mhz = clk[0].split()[0] if clk and clk[0] else ""
        return e0.elapsed_time(e1) / n, (int(mhz) if mhz.isdigit() else None)

    def time_it(run):
        run()
        one, _ = window(run, 3, False)
        n = max(3, int(args.min_ms / max(one, 1e-3)) + 1)
        return window(run, n, True)

    baseline = None
    if args.baseline_lib:
        import ctypes
        baseline = ctypes.CDLL(os.path.abspath(args.baseline_lib))
        baseline.vx_last_error.restype = ctypes.c_char_p
    widths = [int(w) for w in args.widths.split(",")]
    bpf = lambda bn: (128.0 + bn) / (128.0 * bn)
    rows, clocks = [], []
    tot = {"parent": 0.0, "coop": 0.0, "default": 0.0, "best": 0.0}
    for (kind, M, N, K), cnt in shapes:
        gen = torch.Generator(device="cuda").manual_seed(M + 7 * N + 13 * K)
        fl = 2.0 * M * N * K
        geglu = "geglu" in kind
        if kind.startswith(("conv", "upconv")):
            side = int(round((M / FRAMES) ** 0.5))
            if kind == "upconv3x3":
                C = K // 4
                x = torch.randn(FRAMES, side // 2, side // 2, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(4 * N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                make = lambda bn: (lambda: ops.upconv3x3(x, w, bias, block_n=bn))
            elif kind == "conv3x3 s2":
                C = K // 9
                x = torch.randn(FRAMES, 2 * side, 2 * side, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                make = lambda bn: (lambda: ops.conv3x3_s2(x, w, bias, block_n=bn))
            else:
                C = K // 9
                x = torch.randn(FRAMES, side, side, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                res = torch.randn(M, N, device="cuda", generator=gen).bfloat16()   # conv2 of a resnet adds the shortcut
                make = lambda bn: (lambda: ops.conv3x3(x, w, bias, residual=res, block_n=bn))
        else:
            a = torch.randn(M, K, device="cuda", generator=gen).bfloat16()
            w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
            bias = torch.randn(N, device="cuda", generator=gen)
            res = torch.randn(M, N, device="cuda", generator=gen).bfloat16() if kind in RESIDUAL else None

            def make(bn, pack=None):
                if geglu:
                    wp, bp, _ = ops.pack_geglu(w, bias, pack or bn)
                    return lambda: ops.gemm(a, wp, bp, geglu=True, block_n=pack or bn)
                return lambda: ops.gemm(a, w, bias, residual=res, block_n=bn)
        # arm -> (run, env VX_GEMM_PP, library)
        arms = {}
        if baseline is not None:
            arms["parent"] = (make(256) if geglu else make(0), None, baseline)
        arms["coop"] = (make(256) if geglu else make(0), 0, lib)
        for bn in widths:
            if N % bn == 0 and (not geglu or bn % 64 == 0):
                arms[f"pp{bn}"] = (make(bn), 1, lib)
        arms["default"] = (make(0, ops.geglu_block_n(N)) if geglu else make(0), None, lib)

        def use(name):
            _, pp, l = arms[name]
            _ffi._lib = l
            set_env(VX_GEMM_PP=pp)
        info, outs = {}, {}
        for name in arms:
            use(name)
            info[name] = launch_info(arms[name][0])
            outs[name] = arms[name][0]().clone()
        torch.cuda.synchronize()
        same = all(torch.equal(outs["coop"], o) for o in outs.values())
        twin = next((k for k in arms if k not in ("default", "parent") and info[k] == info["default"]), None)
        timed = [k for k in arms if k != "default" or twin is None]
        ms = {k: [] for k in timed}
        for _ in range(args.rounds):
            for name in timed:
                use(name)
                t, clk = time_it(arms[name][0])
                ms[name].append(t)
                clocks += [clk] if clk else []
        _ffi._lib = lib
        set_env(VX_GEMM_PP=None)
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        sp = {k: (max(v) - min(v)) / med[k] for k, v in ms.items()}
        if twin is not None:
            med["default"], sp["default"] = med[twin], sp[twin]
        fastest = min((k for k in med if k not in ("default", "parent")), key=med.get)
        tot["coop"] += med["coop"] * cnt
        tot["default"] += med["default"] * cnt
        tot["best"] += med[fastest] * cnt
        tot["parent"] += med.get("parent", 0.0) * cnt
        row = dict(kind=kind, M=M, N=N, K=K, launches=cnt, geglu=geglu, bit_equal=same, fastest=fastest,
                   default_is=twin or "default",
                   arms={k: dict(bn=info[k][0], pp=info[k][1], rr=info[k][2], ms=med[k], spread=sp[k],
                                 tflops=fl / med[k] / 1e9, bpf=bpf(info[k][0])) for k in med})
        cells = " | ".join(f"{k} bn {info[k][0]}{'pp' if info[k][1] else 'co'}{'r' if info[k][2] else ''} {med[k]:.4f} ms "
                           f"(+-{100 * sp[k]:.1f}%) {fl / med[k] / 1e12:.0f}T" for k in med if k != "default")
        print(f"{kind:12s} {M:7d} {N:6d} {K:6d} | {cells} | default = {twin or 'own'} {med['default']:.4f} ms "
              f"coop/default {med['coop'] / med['default']:.3f} | fastest {fastest} | bit-equal {same}", flush=True)
        rows.append(row)
    mhz = sorted(clocks)[len(clocks) // 2] if clocks else None
    rate = lambda t: f"{t:.2f} ms ({total / t / 1e9:.0f} TFLOP/s)" if t else "not run"
    print(f"one forward, GEMM + conv launches: parent {rate(tot['parent'])}, cooperative {rate(tot['coop'])}, "
          f"default rule {rate(tot['default'])}, fastest arm per shape {rate(tot['best'])}; SM clock {mhz} MHz; {device}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": device, "sm_mhz": mhz, "totals_ms": tot, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
