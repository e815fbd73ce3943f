"""What ptxas made of tc_gemm_kernel (no GPU needed): one full-width wgmma per k16 step, issued back to back.

A function call anywhere in the wgmma k-loop (a printf or assert in a wait, for instance) makes ptxas serialise every
wgmma.mma_async of the kernel: each HGMMA then sits behind its own WARPGROUP.DEPBAR and its whole latency is exposed
(ptxas warning C7510).  These tests read the compiler's own output for every instance tc_gemm_kernel<kNJ>, kNJ = 1..8:
the SASS of the built library and the `-Xptxas -v` log of the build."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from tooncrafter_b200 import build

LOG = build.PKG_DIR / "build" / "build.log"
KERNEL = re.compile(r"tc_gemm_kernelILi(\d)E")


def _built():
    build.build()
    if not LOG.exists():              # library up to date but its log gone: rebuild to get the ptxas report back
        build.build(force=True)
    return build.LIB_PATH


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), str(Path(build._nvcc()).with_name("cuobjdump"))):
        if cand and Path(cand).exists():
            return cand
    return None


def _gemm_sass():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", str(_built())], capture_output=True, text=True, check=True).stdout
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        m = KERNEL.search(body.split("\n", 1)[0])
        if m:
            out[int(m.group(1))] = body
    return out


def test_gemm_issues_one_full_width_wgmma_per_k16_step_without_serialising():
    kernels = _gemm_sass()
    assert sorted(kernels) == list(range(1, 9))
    depbars = set()
    for nj, body in kernels.items():
        shapes = set(re.findall(r"HGMMA\.(\d+x\d+x\d+)", body))
        assert shapes == {f"64x{32 * nj}x16"}, (nj, shapes)
        n_mma = len(re.findall(r"\bHGMMA\.", body))
        n_wait = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body))
        assert n_mma >= 4, (nj, n_mma)           # the four k16 steps of a 64-wide k-block
        # the k-loop's wait for the previous k-block and the final drain: not one wait per instruction
        assert 1 <= n_wait <= 2, (nj, n_mma, n_wait)
        depbars.add(n_wait)
    assert len(depbars) == 1, depbars


def test_gemm_build_log_has_no_serialisation_warning_and_no_spills():
    _built()
    log = LOG.read_text()
    assert "C7510" not in log, [ln for ln in log.splitlines() if "C7510" in ln][:3]
    props = re.findall(r"Function properties for (\S+)\n\s*(.*)", log)
    gemm = {int(KERNEL.search(name).group(1)): line for name, line in props if KERNEL.search(name)}
    assert sorted(gemm) == list(range(1, 9))
    for nj, line in gemm.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (nj, line)
