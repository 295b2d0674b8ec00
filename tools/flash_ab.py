"""A/B timing of the two flash-attention loops on the attention shapes of one UNet forward of the benchmark workload
(b = 2 CFG halves x f = 16 frames, 64x64 latents, 8 heads).

    python tools/flash_ab.py [--launches 50] [--rounds 3] [--baseline-lib LIB] [--plan]

Per shape the arms alternate, A B (C) A B (C), `--rounds` times each:
  old     VX_FA_V1=1, the serial loop of this build;
  parent  (with --baseline-lib: a libvxb200.so built from an earlier commit) that library's default loop;
  new     this build's default loop.
One sample is `--launches` back-to-back launches between two CUDA events.  Prints ms per launch (median over rounds, with
the spread), TFLOP/s by the benchmark's formula 4 B Nq Nk C, the speedup of new over old and over the parent, whether the
outputs are bit-equal, and for hd 40 the share of the exponential bound (a 64x64 score block costs a warpgroup 4096 ex2 at
16 per clock and SM = 256 clocks) at the SM clock sampled during the run.
Inputs come from a seed.  `--plan` prints the shape and FLOP table and stops; timing without a CUDA device is an error."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADS = 8
# (name, Bq, N, hd, kv_div): attn1 over all 32 frames, attn1_5 over the 16 conditional frames against one bank per window
SHAPES = [("attn1   64x64", 32, 4096, 40, 1), ("attn1_5 64x64", 16, 4096, 40, 16),
          ("attn1   32x32", 32, 1024, 80, 1), ("attn1_5 32x32", 16, 1024, 80, 16),
          ("attn1   16x16", 32, 256, 160, 1), ("attn1    8x8 ", 32, 64, 160, 1)]


def flops(Bq, N, hd):
    return 4.0 * Bq * N * N * HEADS * hd


def ex2_bound_ms(Bq, N, sm_mhz, sms):
    """Least time of the softmax exponentials: (N / 64)^2 score blocks per (frame, head), 256 clocks of one SM each."""
    blocks = Bq * HEADS * (N / 64.0) ** 2
    return blocks * 256.0 / sms / (sm_mhz * 1e3)


def smi(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else "unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plan", action="store_true")
    ap.add_argument("--baseline-lib", default=None, help="libvxb200.so of an earlier build, timed as the parent arm")
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()

    print(f"{'shape':14s} {'Bq':>3s} {'N':>5s} {'hd':>4s} {'kv_div':>6s} {'GFLOP':>9s}")
    for name, Bq, N, hd, kv_div in SHAPES:
        print(f"{name:14s} {Bq:3d} {N:5d} {hd:4d} {kv_div:6d} {flops(Bq, N, hd) / 1e9:9.1f}")
    if args.plan:
        return

    import torch
    if not torch.cuda.is_available():
        sys.exit("flash_ab: no CUDA device; timings are only taken on the GPU")
    from vexpress_b200 import _ffi, ops
    _ffi.require_sm90()
    print("device:", smi("name,power.limit,clocks.max.sm"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    lib = _ffi.lib()
    baseline = None
    if args.baseline_lib:
        import ctypes
        baseline = ctypes.CDLL(os.path.abspath(args.baseline_lib))
        baseline.vx_last_error.restype = ctypes.c_char_p
    arms = ["old"] + (["parent"] if baseline is not None else []) + ["new"]

    def use(arm):
        if arm == "old":
            os.environ["VX_FA_V1"] = "1"
        else:
            os.environ.pop("VX_FA_V1", None)
        _ffi._lib = baseline if arm == "parent" else lib
        _ffi._lib.vx_flash_reload_env()

    rows = []
    for name, Bq, N, hd, kv_div in SHAPES:
        C = HEADS * hd
        g = torch.Generator(device="cuda").manual_seed(Bq * N + hd)
        q = torch.randn(Bq * N, C, device="cuda", generator=g).bfloat16()
        kv = torch.randn((Bq // kv_div) * N, 2 * C, device="cuda", generator=g).bfloat16()
        out = torch.empty_like(q)
        run = lambda: ops.flash_attention(q, kv[:, :C], kv[:, C:], HEADS, N, N, kv_div, out=out)
        results = {}
        for arm in arms:
            use(arm)
            for _ in range(5):
                run()
            results[arm] = out.clone()
        torch.cuda.synchronize()
        same = all(torch.equal(results["old"], r) for r in results.values())
        ms = {arm: [] for arm in arms}
        clocks = []
        for _ in range(args.rounds):
            for arm in arms:
                use(arm)
                run()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    run()
                e1.record()
                clk = smi("clocks.sm")   # sampled while the launches are in flight
                e1.synchronize()
                ms[arm].append(e0.elapsed_time(e1) / args.launches)
                if clk.split()[0].isdigit():
                    clocks.append(int(clk.split()[0]))
        use("new")
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        spread = {k: (max(v) - min(v)) / med[k] for k, v in ms.items()}
        mhz = sorted(clocks)[len(clocks) // 2] if clocks else None
        row = {"shape": name.strip(), "Bq": Bq, "N": N, "hd": hd, "kv_div": kv_div, "bit_equal": same, "sm_mhz": mhz}
        line = f"{name:14s}"
        for arm in arms:
            row[f"{arm}_ms"], row[f"{arm}_spread"] = med[arm], spread[arm]
            row[f"{arm}_tflops"] = flops(Bq, N, hd) / med[arm] / 1e9
            line += f" {arm} {med[arm]:8.4f} ms (+-{100 * spread[arm]:4.1f}%) {row[f'{arm}_tflops']:6.1f} TFLOP/s |"
        row["speedup"] = med["old"] / med["new"]
        line += f" new/old x{row['speedup']:.2f}"
        if baseline is not None:
            row["speedup_vs_parent"] = med["parent"] / med["new"]
            line += f" new/parent x{row['speedup_vs_parent']:.2f}"
        line += f" | bit-equal {same} | SM {mhz} MHz"
        if hd == 40 and mhz:
            bound = ex2_bound_ms(Bq, N, mhz, sms)
            line += " | ex2 bound " + f"{bound:.3f} ms:"
            for arm in arms:
                row[f"ex2_bound_share_{arm}"] = bound / med[arm]
                line += f" {arm} {bound / med[arm]:.2f}"
        print(line, flush=True)
        rows.append(row)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": smi("name,power.limit,clocks.max.sm"), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
