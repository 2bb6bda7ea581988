"""CPU tier: the SASS of the tensor-core conv kernels (styletts2_b200/csrc/conv_tc.cu) has the 128-frame tile shape and the
per-warpgroup register budgets, no GPU needed.

Channel-major kernels give each consumer warpgroup 64 output channels x 128 frames (m64n128 MMAs, K = 16 fp16, K = 32 e4m3 for
FAST); time-major kernels give each warpgroup 64 frames x all NC = 2 NH channels (m64n(NC)).  Both need the consumer warpgroups
to take registers from the producer ones (setmaxnreg: USETMAXREG.TRY_ALLOC / DEALLOC)."""
import re

import pytest

from test_cpu_conv_tc_codegen import ALL, _kernel, codegen  # noqa: F401  (module-scoped compile fixture)


def _gmma_shapes(sass):
    """per conv kernel: {(op, N, K)} of the MMAs with fp32 accumulators, and the USETMAXREG forms it contains"""
    shapes, regs, name = {}, {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = _kernel(m.group(1))
            if name:
                shapes[name], regs[name] = set(), set()
            continue
        if not name:
            continue
        m = re.search(r"\b([HQ]GMMA)\.64x(\d+)x(\d+)\.F32", line)
        if m:
            shapes[name].add((m.group(1), int(m.group(2)), int(m.group(3))))
        m = re.search(r"USETMAXREG\.(TRY_ALLOC|DEALLOC)", line)
        if m:
            regs[name].add(m.group(1))
    return shapes, regs


def _expected(kernel):
    m = re.fullmatch(r"(tct?)<(\d+)>", kernel)
    if m.group(1) == "tc":
        ops = {("HGMMA", 128, 16)}
        return ops | {("QGMMA", 128, 32)} if m.group(2) == "0" else ops
    n = 2 * int(m.group(2))
    return {("HGMMA", n, 16), ("QGMMA", n, 32)}


@pytest.mark.parametrize("kernel", ALL)
def test_mma_tile_shape(codegen, kernel):
    shapes, _ = _gmma_shapes(codegen[2])
    assert shapes[kernel] == _expected(kernel), (kernel, sorted(shapes[kernel]))


@pytest.mark.parametrize("kernel", ALL)
def test_warpgroup_register_budgets(codegen, kernel):
    _, regs = _gmma_shapes(codegen[2])
    assert regs[kernel] == {"TRY_ALLOC", "DEALLOC"}, (kernel, regs[kernel])
