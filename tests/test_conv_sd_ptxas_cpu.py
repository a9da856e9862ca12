"""CPU check of what ptxas makes of the shifted-descriptor convolution kernel (csrc/bx_conv_sd.cu), compiled for sm_90a with the
flags of csrc/build.py: no conv_sd_kernel instantiation may have its wgmma chain serialised for lack of registers (C7511), spill,
or keep a stack frame, and in the SASS the HGMMAs of a chunk share one WARPGROUP.DEPBAR instead of waiting one by one.  All of
that depends on the register split between the producer and MMA warpgroups (setmaxnreg) and on no wgmma writing a sub-range
of another in-flight wgmma's accumulator; a change that breaks either shows up here before any GPU run."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "buffer-x_b200", "csrc")


def _build_module():
    spec = importlib.util.spec_from_file_location("_bx_build_flags", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _tool(nvcc, name):
    cand = os.path.join(os.path.dirname(nvcc), name) if os.path.isabs(nvcc) else None
    return cand if cand and os.path.exists(cand) else shutil.which(name)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and shutil.which(nvcc) is None:
        pytest.skip("nvcc not available")
    obj = str(tmp_path_factory.mktemp("conv_sd") / "bx_conv_sd.o")
    cmd = [nvcc] + b.ARCH + b.COMMON + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "bx_conv_sd.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return nvcc, obj, r.stdout + r.stderr


def _kernels(log):
    """{mangled name: text of its ptxas report} for every conv_sd_kernel instantiation."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1) if "conv_sd_kernel" in m.group(1) else None
            if cur:
                out[cur] = ""
        elif cur:
            out[cur] += line + "\n"
    return out


def test_conv_sd_kernels_no_serialised_wgmma_no_spills(compiled):
    _, _, log = compiled
    kernels = _kernels(log)
    assert len(kernels) == 12, f"expected the 12 conv_sd_kernel instantiations (Cout 32/64/128 x input x output), got {len(kernels)}"
    serialised = [ln for ln in log.splitlines() if "C7511" in ln and "conv_sd_kernel" in ln]
    assert not serialised, "wgmma serialised:\n" + "\n".join(serialised)
    for name, rep in kernels.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
        assert m, f"no stack/spill line for {name}:\n{rep}"
        assert m.groups() == ("0", "0", "0"), f"{name}: {m.group(0)}"
        # the setmaxnreg split (SdCfg::PROD_REGS / MMA_REGS) hands out exactly 384 x 168 registers: the launch allocation
        m = re.search(r"Used (\d+) registers", rep)
        assert m and m.group(1) == "168", f"{name}: launch allocation {m.group(1) if m else '?'} registers, the split assumes 168"


def test_conv_sd_hgmma_chain_not_serialised_in_sass(compiled):
    nvcc, obj, _ = compiled
    cuobjdump = _tool(nvcc, "cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    r = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    counts, name = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "conv_sd_kernel" in m.group(1) else None
            if name:
                counts[name] = [0, 0]
        elif name:
            counts[name][0] += "HGMMA" in line
            counts[name][1] += "WARPGROUP.DEPBAR" in line
    assert len(counts) == 12
    for name, (hgmma, depbar) in counts.items():
        # one wait per accumulator pass over a chunk (1, or 2 for the two-pass Cout 128 fp32-input form), not one per HGMMA
        assert hgmma >= 27 and depbar <= 2, f"{name}: {hgmma} HGMMA, {depbar} WARPGROUP.DEPBAR"
