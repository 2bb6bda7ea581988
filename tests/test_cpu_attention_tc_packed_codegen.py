"""CPU tier: what ptxas makes of the packed-row instantiation of the tensor-core attention kernel
(styletts2_b200/csrc/attention_tc.cu, attention_tc_kernel<true>, st2_attention_tc_packed), no GPU needed.

The packed instantiation issues the same wgmma shapes as the padded one (m64n128k16 for S = QK^T, m64n64k16 for O = PV,
fp32 accumulators), and adding it left the padded kernel's instructions exactly as they were: tests/golden/
attention_tc_sass.json holds the instruction count and hash of attention_tc_kernel before the packed path existed."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

from styletts2_b200 import build

SRC = os.path.join(build.CSRC, "attention_tc.cu")
CUOBJDUMP = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_tc_sass.json")

pytestmark = pytest.mark.skipif(not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)), reason="nvcc not available")


def _instantiation(mangled):
    """mangled entry name -> 'padded' / 'packed' for the attention kernel, None otherwise"""
    m = re.search(r"attention_tc_kernelILb([01])E", mangled)
    return None if not m else ("packed" if m.group(1) == "1" else "padded")


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("attention_tc_codegen") / "attention_tc.o")
    p = subprocess.run([build.NVCC, *build.FLAGS, "-c", SRC, "-o", obj], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    text = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = _instantiation(m.group(1))
            if name:
                funcs[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if name and m:
            funcs[name].append(m.group(1))          # the instruction text: no address, no encoding
    assert sorted(funcs) == ["packed", "padded"], sorted(funcs)
    return funcs


def _shapes(instrs):
    return sorted({m.group(0) for i in instrs for m in [re.search(r"\bHGMMA\.64x\d+x\d+\.F32", i)] if m})


def test_packed_issues_the_same_wgmma_shapes(sass):
    assert _shapes(sass["packed"]) == _shapes(sass["padded"]) == ["HGMMA.64x128x16.F32", "HGMMA.64x64x16.F32"]
    count = lambda instrs: sum(1 for i in instrs if "HGMMA." in i)         # noqa: E731
    assert count(sass["packed"]) == count(sass["padded"])


def test_padded_kernel_unchanged(sass):
    ref = json.load(open(FIXTURE))
    ver = subprocess.run([build.NVCC, "--version"], capture_output=True, text=True).stdout
    if ref["nvcc_release"] not in ver:
        pytest.skip(f"the fixture was recorded with nvcc {ref['nvcc_release']}")
    got = sass["padded"]
    assert len(got) == ref["instructions"]
    assert hashlib.sha256("\n".join(got).encode()).hexdigest() == ref["sha256"]
