"""A/B timing of the three GroupNorm kernels (cluster-resident, one-launch rendezvous, statistics + apply pair) between this
tree's library and a baseline library built from an earlier commit, at the distinct GroupNorm shapes of one UNet forward of
the benchmark workload (b = 2 CFG halves x f = 16 frames, 64x64 latents: 32 frames per launch) and of the VAE decoder at
512 x 512 (one frame per launch).

    python tools/norm_ab.py --baseline-lib LIB [--min-ms 200] [--rounds 5] [--json FILE]

Both libraries are loaded into one process and called through the same C entry points with the same operands, the
workspace sized and S chosen as ops.groupnorm does from each library's own capacity query.  Where a library's one-launch
kernel declines (the grid would not be co-resident) its ``fused`` arm runs the statistics + apply pair, as ops.groupnorm
does, and the row is marked.  Per shape and path the two arms alternate, arm by arm, ``--rounds``
times; one sample is as many back-to-back launches as fill at least ``--min-ms`` between two CUDA events.  Prints ms per
launch (median over rounds, with the spread) and the new / baseline ratio, per path the sum over the shapes,
and the card name and power limit read in the same run.  The cluster arm is timed where the frame fits a cluster (the
library returns 2 elsewhere).  Inputs come from a seed; timing without a CUDA device is an error."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (NB, HW, C1, C2, silu): the distinct GroupNorm shapes of the two workloads
UNET = [(32, 4096, 320, 0, True), (32, 4096, 320, 320, True), (32, 4096, 640, 320, True),
        (32, 4096, 320, 0, False), (32, 1024, 320, 0, True), (32, 1024, 640, 0, True),
        (32, 1024, 640, 320, True), (32, 1024, 640, 640, True), (32, 1024, 1280, 640, True),
        (32, 1024, 640, 0, False), (32, 256, 640, 0, True), (32, 256, 1280, 0, True),
        (32, 256, 1280, 640, True), (32, 256, 1280, 1280, True), (32, 256, 1280, 0, False),
        (32, 64, 1280, 0, True), (32, 64, 1280, 1280, True), (32, 64, 1280, 0, False)]
VAE = [(1, 4096, 512, 0, True), (1, 4096, 512, 0, False), (1, 16384, 512, 0, True),
       (1, 65536, 512, 0, True), (1, 65536, 256, 0, True), (1, 262144, 256, 0, True),
       (1, 262144, 128, 0, True)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", required=True)
    ap.add_argument("--min-ms", type=float, default=200.0)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("norm_ab: no CUDA device")
    from vexpress_b200 import _ffi
    from vexpress_b200._ffi import c_float, c_int, c_ll, ptr
    _ffi.require_sm90()
    libs = {"new": _ffi.lib(), "base": ctypes.CDLL(os.path.abspath(args.baseline_lib))}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}")
    st = torch.cuda.current_stream()
    sp = ctypes.c_void_p(st.cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows, totals = [], {}
    for group, shapes in (("unet", UNET), ("vae", VAE)):
        for NB, HW, C1, C2, silu in shapes:
            C = C1 + C2
            x1 = torch.randn(NB * HW, C1, device="cuda", generator=g).bfloat16()
            x2 = torch.randn(NB * HW, C2, device="cuda", generator=g).bfloat16() if C2 else None
            gam = 1 + 0.1 * torch.randn(C, device="cuda", generator=g)
            bet = 0.1 * torch.randn(C, device="cuda", generator=g)
            out = torch.empty(NB * HW, C, device="cuda", dtype=torch.bfloat16)
            Ss = {k: max(1, min(HW // 32, max(int(L.vx_groupnorm_capacity(c_int(C))), 1) // NB, 64)) for k, L in libs.items()}
            ws = torch.empty(NB * 64 * 32 * 3, device="cuda", dtype=torch.float32)
            cnt = torch.zeros(max(2 * NB, 1024), device="cuda", dtype=torch.int32)
            head = (ptr(x1), c_ll(x1.stride(0)), c_int(C1), ptr(x2), c_ll(0 if x2 is None else x2.stride(0)), c_int(C2),
                    c_int(NB), c_int(HW), c_int(32))
            tail = (ptr(gam), ptr(bet), c_float(1e-5), c_int(int(silu)), ptr(out), c_ll(out.stride(0)), sp)

            def launch(arm, path):
                L, S = libs[arm], Ss[arm]
                if path == "cluster":
                    return L.vx_groupnorm_cluster(*head, *tail)
                if path == "fused" and arm not in declined:
                    return L.vx_groupnorm_fused(*head, c_int(S), ptr(ws), ptr(cnt), *tail)
                rc = L.vx_groupnorm_stats(*head, c_int(S), ptr(ws), sp)
                return rc or L.vx_groupnorm_apply(*head, c_int(S), ptr(ws), *tail)

            for path in ("cluster", "fused", "pair"):
                declined = set()
                rcs = {k: launch(k, path) for k in libs}
                torch.cuda.synchronize()
                if path == "cluster" and any(rcs.values()):
                    assert rcs["new"] == rcs["base"] == 2, (path, rcs)
                    continue
                declined = {k for k, rc in rcs.items() if rc == 2}
                assert all(launch(k, path) == 0 for k in libs), (path, rcs)
                t = {"new": [], "base": []}
                reps = {}
                for _ in range(args.rounds):
                    for arm in libs:
                        n = reps.get(arm, 4)
                        while True:
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            for _ in range(n):
                                launch(arm, path)
                            e1.record()
                            e1.synchronize()
                            ms = e0.elapsed_time(e1)
                            if ms >= args.min_ms or arm in reps:
                                break
                            n = max(n * 2, int(n * args.min_ms / max(ms, 1e-3)) + 1)
                        reps[arm] = n
                        t[arm].append(ms / n)
                med = {k: statistics.median(v) for k, v in t.items()}
                spread = {k: (max(v) - min(v)) / med[k] for k, v in t.items()}
                S = "/".join(str(Ss[k]) for k in libs)
                mark = "".join(f" ({k}: pair)" for k in sorted(declined))
                r = dict(group=group, NB=NB, HW=HW, C1=C1, C2=C2, silu=silu, path=path + mark, S=S,
                         new_ms=med["new"], base_ms=med["base"], new_spread=spread["new"], base_spread=spread["base"],
                         ratio=med["new"] / med["base"])
                rows.append(r)
                key = (group, path)
                a, b = totals.get(key, (0.0, 0.0))
                totals[key] = (a + med["new"], b + med["base"])
                print(f"{group:4s} NB {NB:2d} HW {HW:6d} C {C1:4d}+{C2:4d} silu {int(silu)} {path:7s} S {S:5s}: "
                      f"new {1e3 * med['new']:8.2f} us (+-{50 * spread['new']:.1f} %)  base {1e3 * med['base']:8.2f} us "
                      f"(+-{50 * spread['base']:.1f} %)  new/base {r['ratio']:.3f}{mark}", flush=True)
    for (group, path), (a, b) in sorted(totals.items()):
        print(f"sum over the {group} shapes, {path:7s}: new {a:.3f} ms  base {b:.3f} ms  new/base {a / b:.3f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, rows=rows, totals={f"{g_} {p}": v for (g_, p), v in totals.items()}), f, indent=1)


if __name__ == "__main__":
    main()
