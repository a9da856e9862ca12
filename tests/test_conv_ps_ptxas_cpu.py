"""CPU check of what ptxas makes of the per-sample descriptor convolution (csrc/bx_conv_ps.cu), compiled for sm_90a with the
flags of csrc/build.py: no conv_ps_kernel instantiation may spill, keep a stack frame or have its wgmma chain serialised
(C7511); the launch allocation is the 168 registers the setmaxnreg split assumes; the only wgmma widths are the 152-row sample
(Cout <= 32) and its two passes of 80 + 72 rows (Cout >= 64); and each N pass over a chunk has one WARPGROUP.DEPBAR."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "buffer-x_b200", "csrc")


def _build_module():
    spec = importlib.util.spec_from_file_location("_bx_build_flags_ps", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and shutil.which(nvcc) is None:
        pytest.skip("nvcc not available")
    obj = str(tmp_path_factory.mktemp("conv_ps") / "bx_conv_ps.o")
    r = subprocess.run([nvcc] + b.ARCH + b.COMMON + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "bx_conv_ps.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return nvcc, obj, r.stdout + r.stderr


def test_conv_ps_kernels_no_spills_no_serialised_wgmma(compiled):
    _, _, log = compiled
    reports, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if "conv_ps_kernel" in m.group(1) else None
            if cur:
                reports[cur] = ""
        elif cur:
            reports[cur] += line + "\n"
    assert len(reports) == 6, f"expected 6 conv_ps_kernel instantiations (Cout 32/64/128 x output format), got {len(reports)}"
    assert not [ln for ln in log.splitlines() if "C7511" in ln], "wgmma serialised"
    for name, rep in reports.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
        assert m and m.groups() == ("0", "0", "0"), f"{name}: {m.group(0) if m else rep}"
        m = re.search(r"Used (\d+) registers", rep)
        assert m and m.group(1) == "168", f"{name}: launch allocation {m.group(1) if m else '?'}"


def test_conv_ps_hgmma_widths_and_waits(compiled):
    nvcc, obj, _ = compiled
    cand = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else None
    cuobjdump = cand if cand and os.path.exists(cand) else shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    r = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    stats, name = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "conv_ps_kernel" in m.group(1) else None
            if name:
                stats[name] = [set(), 0, 0]
        elif name:
            m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
            if m:
                stats[name][0].add(m.group(1))
                stats[name][1] += 1
            stats[name][2] += "WARPGROUP.DEPBAR" in line
    assert len(stats) == 6
    for name, (shapes, hgmma, depbar) in stats.items():
        nt = int(re.search(r"conv_ps_kernelILi(\d+)E", name).group(1))
        if nt == 32:      # P * ah, Q * al per tap: 18 HGMMAs, one pass
            assert shapes == {"64x152x16"} and hgmma == 18 and depbar == 1, (name, shapes, hgmma, depbar)
        else:             # three per tap, two passes
            assert shapes == {"64x80x16", "64x72x16"} and hgmma == 54 and depbar == 2, (name, shapes, hgmma, depbar)
