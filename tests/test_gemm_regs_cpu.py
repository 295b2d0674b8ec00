"""The GEMM kernel's register split takes effect: every gemm_wgmma_kernel instantiation keeps its setmaxnreg instructions
and spills nothing.

gemm_wgmma_kernel gives the producer warpgroup 40 registers per thread and the two consumer warpgroups 232 (setmaxnreg).
When ptxas cannot honour that split it drops the instructions with warning C7507 (or C7512), and the consumers run with
the 168 registers that 384 threads launch with: the wide tiles then spill their accumulators.  This test compiles
vx_gemm.cu for sm_90a as build.sh does, with -Xptxas -v, into a temporary directory (no GPU needed)."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
CSRC = os.path.join(ROOT, "v-express_b200", "csrc")


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.check_call([sys.executable, os.path.join(CSRC, "gen_wgmma.py"), os.path.join(tmp, "vx_wgmma_gen.cuh")])
        obj = os.path.join(tmp, "vx_gemm.o")
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                            "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
                            "-I" + os.path.join(ROOT, "include"), "-I" + tmp, "-c", os.path.join(CSRC, "vx_gemm.cu"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _per_kernel_ptxas(log):
    """{mangled gemm_wgmma_kernel name: ptxas lines about it}"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(_ZN2vx17gemm_wgmma_kernel\w+)", line)
        if m:
            out.setdefault(m.group(1), [])
        if "Compiling entry function" in line or "Function properties for" in line:
            cur = m.group(1) if m else None
        if cur:
            out[cur].append(line)
        if m and re.search(r"C75(07|12)", line):
            out[m.group(1)].append(line)
    return out


def test_every_instantiation_keeps_setmaxnreg_and_does_not_spill(compiled):
    log, sass = compiled
    kernels = _per_kernel_ptxas(log)
    assert len(kernels) >= 21, sorted(kernels)   # 8 cooperative + 8 LayerNorm + 5 ping-pong widths
    dropped = re.findall(r".*C75(?:07|12).*gemm_wgmma_kernel.*", log)
    assert not dropped, "\n".join(dropped)
    spills = {k: l for k, ls in kernels.items() for l in ls
              if re.search(r"[1-9]\d* bytes spill (stores|loads)", l)}
    assert not spills, spills
    funcs = re.split(r"\n\s*Function : ", sass)
    with_setmaxnreg = {f.split()[0] for f in funcs[1:] if "USETMAXREG" in f}
    missing = sorted(k for k in kernels if k not in with_setmaxnreg)
    assert not missing, missing
