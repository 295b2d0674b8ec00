"""A/B timing of the two GEMM consumer schedules (cooperative vs ping-pong) on the GEMM / convolution shapes of one UNet
forward of the benchmark workload (b = 2 CFG halves x f = 16 frames, 64x64 latents: 32 frames per launch).

    python tools/gemm_ab.py [--min-ms 300] [--rounds 3] [--plan] [--json FILE]

The shape list restates the launches `UNetEngine.forward_frames` issues (4 down levels of 320 / 640 / 1280 / 1280 channels,
the mid block, 4 up levels with 3 resnets each; spatial transformers at the 64 / 32 / 16 levels, motion modules
everywhere).  Per plain-GEMM shape three arms alternate, A B C A B C, `--rounds` times each:
  old   cooperative schedule (VX_GEMM_PP=0) at the column tile the library picks for it;
  new   ping-pong schedule (VX_GEMM_PP=1) at the column tile the library picks for it (<= 96);
  same  cooperative schedule at the ping-pong arm's column tile: the same 128 x bn tile, operand traffic and accumulators
        per thread as `new`, so new against same isolates the schedule, old against same the tile width.
One sample is as many back-to-back launches as fill at least `--min-ms` between two CUDA events; the SM clock is read by a
thread while that window runs.  GEGLU weights are packed for each arm's tile.  Prints ms per launch (median over rounds,
with the spread), TFLOP/s (2 M N K), the L2 -> shared-memory operand bytes per FLOP of the tile ((128 + bn) / (128 bn):
every K block moves a 128-row A box and a bn-row W box), the ratios, which schedule the default rule picks, and whether
the outputs are bit-identical.  The convolutions have one schedule (cooperative) and are timed once per round.  The card
name, power limit and the median sampled SM clock are printed with the table.  Inputs come from a seed.
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
        lib.vx_gemm_reload_env()

    def launch_info(run):
        """(bn, pp) of one launch, from the VX_GEMM_VERBOSE log on fd 2"""
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
        m = re.findall(r"bn=(\d+) pp=(\d+)", log)
        return (int(m[-1][0]), int(m[-1][1])) if m else (0, 0)

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

    bpf = lambda bn: (128.0 + bn) / (128.0 * bn)
    rows, clocks = [], []
    tot = {"old": 0.0, "new": 0.0, "default": 0.0}
    for (kind, M, N, K), cnt in shapes:
        gen = torch.Generator(device="cuda").manual_seed(M + 7 * N + 13 * K)
        fl = 2.0 * M * N * K
        conv = kind.startswith("conv") or kind.startswith("upconv")
        if conv:
            side = int(round((M / FRAMES) ** 0.5))
            if kind == "upconv3x3":
                C = K // 4
                x = torch.randn(FRAMES, side // 2, side // 2, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(4 * N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                run = lambda: ops.upconv3x3(x, w, bias)
            elif kind == "conv3x3 s2":
                C = K // 9
                x = torch.randn(FRAMES, 2 * side, 2 * side, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                run = lambda: ops.conv3x3_s2(x, w, bias)
            else:
                C = K // 9
                x = torch.randn(FRAMES, side, side, C, device="cuda", generator=gen).bfloat16()
                w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
                bias = torch.randn(N, device="cuda", generator=gen)
                run = lambda: ops.conv3x3(x, w, bias)
            bn, _ = launch_info(run)
            ms = []
            for _ in range(args.rounds):
                t, clk = time_it(run)
                ms.append(t)
                clocks += [clk] if clk else []
            med = sorted(ms)[len(ms) // 2]
            for k in tot:
                tot[k] += med * cnt
            row = dict(kind=kind, M=M, N=N, K=K, launches=cnt, sched="cooperative only", old_bn=bn, old_ms=med,
                       old_spread=(max(ms) - min(ms)) / med, old_tflops=fl / med / 1e9, old_bpf=bpf(bn))
            print(f"{kind:12s} {M:7d} {N:6d} {K:6d} | coop bn {bn:3d} {med:8.4f} ms {row['old_tflops']:6.1f} TFLOP/s "
                  f"{bpf(bn):.4f} B/FLOP | (one schedule)", flush=True)
            rows.append(row)
            continue
        geglu = "geglu" in kind
        a = torch.randn(M, K, device="cuda", generator=gen).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
        bias = torch.randn(N, device="cuda", generator=gen)
        res = torch.randn(M, N, device="cuda", generator=gen).bfloat16() if kind in RESIDUAL else None
        arms = {}

        def arm(pp, bn=0):
            if geglu:
                gbn = bn or (64 if pp == 1 else ops.geglu_block_n(N))
                wp, bp, _ = ops.pack_geglu(w, bias, gbn)
                return lambda: ops.gemm(a, wp, bp, geglu=True, block_n=gbn)
            return lambda: ops.gemm(a, w, bias, residual=res, block_n=bn)
        for name, pp in (("old", 0), ("new", 1), ("default", None)):
            set_env(VX_GEMM_PP=pp)
            run = arm(pp)
            arms[name] = (run, launch_info(run), pp)
        nbn = arms["new"][1][0]
        set_env(VX_GEMM_PP=0)
        run = arm(0, nbn)
        arms["same"] = (run, launch_info(run), 0)
        outs = {}
        for name, (run, _, pp) in arms.items():
            set_env(VX_GEMM_PP=pp)
            outs[name] = run()
        torch.cuda.synchronize()
        same = all(torch.equal(outs["old"], o) for o in outs.values())
        timed = ("old", "new", "same")
        ms = {k: [] for k in timed}
        for _ in range(args.rounds):
            for name in timed:
                run, _, pp = arms[name]
                set_env(VX_GEMM_PP=pp)
                t, clk = time_it(run)
                ms[name].append(t)
                clocks += [clk] if clk else []
        set_env(VX_GEMM_PP=None)
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        sp = {k: (max(v) - min(v)) / med[k] for k, v in ms.items()}
        (obn, _), (nbn, npp), (dbn, dpp), (sbn, spp) = (arms[k][1] for k in ("old", "new", "default", "same"))
        dflt = "new" if dpp else "same" if dbn == sbn and dbn != obn else "old"
        tot["old"] += med["old"] * cnt
        tot["new"] += med["new"] * cnt
        tot["default"] += med[dflt] * cnt
        row = dict(kind=kind, M=M, N=N, K=K, launches=cnt, geglu=geglu, bit_equal=same, old_bn=obn, new_bn=nbn,
                   new_is_pp=bool(npp), same_bn=sbn, default_bn=dbn, default_pp=bool(dpp),
                   **{f"{k}_ms": med[k] for k in timed}, **{f"{k}_spread": sp[k] for k in timed},
                   **{f"{k}_tflops": fl / med[k] / 1e9 for k in timed}, old_bpf=bpf(obn), new_bpf=bpf(nbn),
                   old_over_new=med["old"] / med["new"], same_over_new=med["same"] / med["new"])
        print(f"{kind:12s} {M:7d} {N:6d} {K:6d} | coop bn {obn:3d} {med['old']:8.4f} ms (+-{100 * sp['old']:4.1f}%) "
              f"{row['old_tflops']:6.1f} TFLOP/s {bpf(obn):.4f} B/FLOP | pp bn {nbn:3d}{'' if npp else ' (coop)'} "
              f"{med['new']:8.4f} ms (+-{100 * sp['new']:4.1f}%) {row['new_tflops']:6.1f} TFLOP/s {bpf(nbn):.4f} B/FLOP | "
              f"coop bn {sbn:3d} {med['same']:8.4f} ms (+-{100 * sp['same']:4.1f}%) | old/new {row['old_over_new']:.3f} "
              f"same/new {row['same_over_new']:.3f} | default {'pp' if dpp else 'coop'} bn {dbn} | bit-equal {same}",
              flush=True)
        rows.append(row)
    mhz = sorted(clocks)[len(clocks) // 2] if clocks else None
    print(f"one forward, GEMM + conv launches: cooperative {tot['old']:.2f} ms ({total / tot['old'] / 1e9:.0f} TFLOP/s), "
          f"ping-pong where available {tot['new']:.2f} ms ({total / tot['new'] / 1e9:.0f} TFLOP/s), "
          f"default rule {tot['default']:.2f} ms ({total / tot['default'] / 1e9:.0f} TFLOP/s); SM clock {mhz} MHz; {device}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": device, "sm_mhz": mhz, "totals_ms": tot, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
