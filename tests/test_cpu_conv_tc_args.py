"""CPU tier: st2_conv1d_tc rejects output layouts its kernels do not write, no GPU needed.

The tensor-core conv kernels store contiguous output positions only: a strided / offset output (y_tstride, y_toffset) and
the reflection duplicate (dup_q0_to) are the SIMT conv's.  The entry point checks its arguments before any CUDA call, so
dummy device pointers are enough to see the rejections."""
import ctypes as C

import pytest

from styletts2_b200 import lib as L


def _args(**over):
    a = L.ConvArgs()
    dummy = C.c_void_p(0x1000)
    a.x, a.y, a.x_bstride, a.y_bstride = dummy, dummy, 256 * 512, 256 * 512
    a.Cin, a.Cout, a.Lin, a.Lq, a.y_len = 256, 256, 512, 512, 512
    a.y_tstride, a.y_toffset = 1, 0
    a.B, a.K, a.stride, a.dil, a.pad = 1, 3, 1, 1, 1
    a.out_div, a.accum_div = 1.0, 1.0
    a.dup_q0_to = -1
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,msg", [
    (dict(y_tstride=2), "contiguous"),
    (dict(y_toffset=1), "contiguous"),
    (dict(dup_q0_to=0), "reflection duplicate"),
])
def test_conv1d_tc_rejects_strided_output_and_reflection_duplicate(lib_built, over, msg):
    a = _args(**over)
    n0 = L.launch_count()
    with pytest.raises(RuntimeError, match=msg):
        L.call("st2_conv1d_tc", C.byref(a), C.c_void_p(0x2000), L.TC_FAST, 0, None)
    assert L.launch_count() == n0
