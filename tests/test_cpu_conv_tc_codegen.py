"""CPU tier: what ptxas makes of the tensor-core conv kernels (styletts2_b200/csrc/conv_tc.cu), no GPU needed.

The consumer warpgroups' wgmmas only overlap (one commit group per weight stage in flight, the f16 and the e4m3 MMA of a
tap back to back) when ptxas can prove the role dispatch warp-uniform.  When it cannot, it reports C7520 ("wgmma ... serialized
due to ... WG.AR in divergent path") and drains the tensor pipe after every MMA (`WARPGROUP.DEPBAR.LE gsb0, 0x0`), which
leaves most of the tensor-core time idle.  The same change decides whether the kernels spill at their 96-register cap."""
import os
import re
import shutil
import subprocess

import pytest

from styletts2_b200 import build

SRC = os.path.join(build.CSRC, "conv_tc.cu")
CUOBJDUMP = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
# tc<recipe> = conv1d_tc_kernel<ST2_TC_FAST / ACCURATE / F16X3>, tct<NH> = conv1d_tct_kernel<NH>
ALL = ["tc<0>", "tc<1>", "tc<2>", "tct<8>", "tct<16>", "tct<32>", "tct<48>", "tct<64>"]
ACCURATE_MAX_SPILL = (56, 108)   # (stores, loads) in bytes of tc<1>: its two accumulators of 32 registers each

pytestmark = pytest.mark.skipif(not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)), reason="nvcc not available")


def _kernel(mangled):
    """mangled entry name -> 'tc<mode>' / 'tct<NH>' for the conv kernels, None otherwise"""
    m = re.search(r"conv1d_(tct?)_kernelILi(\d+)E", mangled)
    return f"{m.group(1)}<{m.group(2)}>" if m else None


@pytest.fixture(scope="module")
def codegen(tmp_path_factory):
    out = tmp_path_factory.mktemp("conv_tc_codegen")
    obj = str(out / "conv_tc.o")
    p = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", obj], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    log = p.stdout + p.stderr
    spills, current = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            current = _kernel(m.group(1))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            spills[current] = (int(m.group(1)), int(m.group(2)))
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return log, spills, sass


def _mma_events(sass):
    """per conv kernel: the sequence of GMMAs ('G') and warpgroup waits ('W<n>') in address order"""
    ev, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = _kernel(m.group(1))
            if name:
                ev[name] = []
            continue
        if not name:
            continue
        if re.search(r"\b[HQ]GMMA\.", line):
            ev[name].append("G")
        else:
            m = re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", line)
            if m:
                ev[name].append("W" + m.group(1))
    return ev


def test_no_serialized_wgmma_warning(codegen):
    log, spills, _ = codegen
    assert sorted(spills) == sorted(ALL), sorted(spills)
    bad = [line for line in log.splitlines() if "C7520" in line and "conv1d_tc" in line]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("kernel", [k for k in ALL if k != "tc<1>"])
def test_no_spills(codegen, kernel):
    """(spill stores, spill loads) in bytes at the 96-register cap of 608 threads per SM"""
    assert codegen[1][kernel] == (0, 0), codegen[1][kernel]


def test_accurate_spills_bounded(codegen):
    st, ld = codegen[1]["tc<1>"]
    assert st <= ACCURATE_MAX_SPILL[0] and ld <= ACCURATE_MAX_SPILL[1], (st, ld)


@pytest.mark.parametrize("kernel", ALL)
def test_mma_pipeline_not_drained(codegen, kernel):
    """No GMMA is followed by a full drain before the next GMMA, and the tap loop waits with one group in flight.  The full
    wait at the end of a tile comes after the loop's `gsb0, 0x1` wait, so it never directly follows a GMMA."""
    ev = _mma_events(codegen[2])[kernel]
    assert ev.count("G") >= 2, ev
    drained = sum(1 for a, b in zip(ev, ev[1:]) if a == "G" and b == "W0x0")
    assert drained == 0, ev
    assert "W0x1" in ev, ev
