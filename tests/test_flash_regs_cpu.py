"""The pipelined flash-attention kernel's register split takes effect: every flash_attn_pipe_kernel instantiation keeps its
setmaxnreg instructions and spills nothing.

flash_attn_pipe_kernel gives the producer warpgroup 24 registers per thread and the consumer warpgroups what is left of
the launch allocation: 160 with three consumers (hd <= 56, two S register sets), 232 with two consumers (hd 80, 160) or
one consumer and two CTAs per SM.  When ptxas cannot honour that split it drops the instructions with warning C7507 (or
C7512), and the consumers run with what the launch gave them: the accumulators then spill.  The test also requires that
no wgmma is serialised (C7513), which ptxas does to the whole kernel when it cannot prove that the two-set schedule
leaves registers alone while their MMA is in flight.  This test compiles vx_flash_attn.cu for sm_90a as build.sh does,
with -Xptxas -v, into a temporary directory (no GPU needed)."""
import os
import re
import subprocess
import sys
import tempfile

import pytest

from test_gemm_regs_cpu import CSRC, ROOT, _nvcc

KERNEL = "_ZN2vx22flash_attn_pipe_kernel"


@pytest.fixture(scope="module")
def compiled():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.check_call([sys.executable, os.path.join(CSRC, "gen_wgmma.py"), os.path.join(tmp, "vx_wgmma_gen.cuh")])
        obj = os.path.join(tmp, "vx_flash_attn.o")
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                            "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
                            "-I" + os.path.join(ROOT, "include"), "-I" + tmp, "-c", os.path.join(CSRC, "vx_flash_attn.cu"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _per_kernel_ptxas(log):
    """{mangled flash_attn_pipe_kernel name: ptxas lines about it}"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(" + KERNEL + r"\w+)", line)
        if m:
            out.setdefault(m.group(1), [])
        if "Compiling entry function" in line or "Function properties for" in line:
            cur = m.group(1) if m else None
        if cur:
            out[cur].append(line)
    return out


def test_every_pipe_instantiation_keeps_setmaxnreg_and_does_not_spill(compiled):
    log, sass = compiled
    kernels = _per_kernel_ptxas(log)
    widths = {(int(h), int(n)) for h, n in (re.search(r"ILi(\d+)ELi(\d+)E", k).groups() for k in kernels)}
    # hd 8 .. 56 with one and three consumer warpgroups, hd 80 and 160 with one and two
    assert widths == ({(h, n) for h in (8, 16, 24, 32, 40, 48, 56) for n in (1, 3)} |
                      {(h, n) for h in (80, 160) for n in (1, 2)}), sorted(widths)
    # a wgmma serialised (C7513 / C7512) would undo the overlap the loop is built for
    serial = re.findall(r".*C75(?:12|13).*flash_attn_pipe_kernel.*", log)
    assert not serial, "\n".join(serial)
    dropped = re.findall(r".*C75(?:07|12).*flash_attn_pipe_kernel.*", log)
    assert not dropped, "\n".join(dropped)
    spills = {k: l for k, ls in kernels.items() for l in ls
              if re.search(r"[1-9]\d* bytes (spill (stores|loads)|stack frame)", l)}
    assert not spills, spills
    funcs = re.split(r"\n\s*Function : ", sass)
    with_setmaxnreg = {f.split()[0] for f in funcs[1:] if "USETMAXREG" in f}
    missing = sorted(k for k in kernels if k not in with_setmaxnreg)
    assert not missing, missing
