"""Register budget of the kNN matcher, from ptxas (no GPU needed): the default k_match_knn<5|10> instance fits 72 registers with no
spill and no stack frame, so that three of its 256-thread CTAs and one 64-thread k_eval_candidate block share an SM's 65536
registers (the speculative schedule runs the candidate evaluation next to the matcher).  The MLOAM_KNN_MB=2 instance and the
instrumented one are compiled from the same body and must not spill either."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "m-loam_b200", "csrc")
NVCC = "/usr/local/cuda/bin/nvcc"
# m-loam_b200/Makefile's NVFLAGS
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-O2", "-Xptxas", "-v"]
SM_REGS = 65536


def _ptxas(src, tmp_path):
    """{demangled entry name: (registers, stack frame B, spill stores B, spill loads B)} of the kernels in csrc/<src>."""
    log = subprocess.run([NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         capture_output=True, text=True, check=True).stderr
    out, cur, frame = {}, None, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            frame = tuple(int(x) for x in m.groups())
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur and frame:
            out[cur] = (int(m.group(1)),) + frame
            cur, frame = None, None
    return out


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("c++filt") is None, reason="needs nvcc and c++filt")
def test_match_knn_register_budget(tmp_path):
    knn = _ptxas("match_kernels.cu", tmp_path)
    ev = [v for k, v in _ptxas("solve_kernels.cu", tmp_path).items() if "k_eval_candidate" in k]
    assert ev, "k_eval_candidate not found in solve_kernels.cu's ptxas log"
    ev_regs = max(v[0] for v in ev)
    for K in (5, 10):
        regs, frame, st, ld = knn[f"void mloam::k_match_knn<{K}>"]
        assert regs <= 72 and frame == 0 and st == 0 and ld == 0, (K, regs, frame, st, ld)
        assert 3 * 256 * regs + 64 * ev_regs <= SM_REGS, (K, regs, ev_regs)
        for stats in ("false", "true"):
            r = knn[f"void mloam::k_match_knn_mb2<{K}, {stats}>"]
            assert r[2] == 0 and r[3] == 0, (K, stats, r)
            assert 2 * 256 * r[0] <= SM_REGS
