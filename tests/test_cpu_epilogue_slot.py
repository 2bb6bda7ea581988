"""CPU tier: the epilogue transpose slot of the tensor-core conv kernels (csrc/conv_tc.cu slot_index, SLOT_FLOATS), restated
in Python.

Each consumer warpgroup moves one slice of its tile's outputs through 4096 floats of shared memory as [channel][frame] rows:
the fragments go in in the wgmma register order, then each warp reads, combines, stores and writes back whole channel rows
(lane l: frames l + 32 m).  For every slice shape the kernels use, the map must be a bijection onto the slot, both views must
be free of shared-memory bank conflicts, and the slice must fit."""
import pytest

SLOT_FLOATS = 4096   # per consumer warpgroup: SM_SLOT holds two
TN, TP = 128, 64     # frames per tile, frames per statistics partial (= per time-major warpgroup)


def slot_index(r, fr, pitch):
    return r * pitch + (fr ^ ((r & 1) | ((r & 6) << 2)))


def tct_slices(nc):
    """time-major, NC channels: slices of up to 64 channels x 64 frames; fragment float 4 j + q (q = 2 i + c) of lane
    (g, t4) in warp w is frame w * 16 + g + 8 i of channel 8 j + 2 t4 + c"""
    sc = min(nc, 64)
    out = []
    for c0 in range(0, nc, sc):
        def frag(w, lane, j, q, c0=c0):
            g, t4 = lane >> 2, lane & 3
            return 8 * j - c0 + 2 * t4 + (q & 1), w * 16 + g + 4 * (q & 2)
        regs = [(j, q) for j in range(nc // 8) if c0 <= 8 * j < c0 + sc for q in range(4)]
        nr = min(sc, nc - c0) // 4
        out.append((min(sc, nc - c0), TP, frag, regs, [list(range(w * nr, w * nr + nr)) for w in range(4)]))
    return out


def tc_slices():
    """channel-major: one slice per 64-frame half h (64 channels x 64 frames); fragment float 32 h + q of lane (g, t4) in
    warp w is channel w * 16 + g + 8 ((q >> 1) & 1), frame 8 (q >> 2) + 2 t4 + (q & 1) of the half"""
    def frag(w, lane, j, q):
        g, t4 = lane >> 2, lane & 3
        return w * 16 + g + 8 * ((q >> 1) & 1), 8 * (q >> 2) + 2 * t4 + (q & 1)
    regs = [(0, q) for q in range(32)]
    return [(64, TP, frag, regs, [list(range(16 * w, 16 * w + 16)) for w in range(4)]) for _ in range(TN // TP)]


SHAPES = [(f"tct nc{nc}", s) for nc in (16, 32, 64, 96, 128) for s in tct_slices(nc)] + [("tc", s) for s in tc_slices()]


@pytest.mark.parametrize("name,shape", SHAPES, ids=[f"{n}-{i}" for i, (n, _) in enumerate(SHAPES)])
def test_slot_map(name, shape):
    rows, pitch, frag, regs, warp_rows = shape
    # fits, and the map is a bijection of the slice's (channel, frame) pairs onto [0, rows * pitch)
    assert rows * pitch <= SLOT_FLOATS, name
    idx = {slot_index(r, fr, pitch): (r, fr) for r in range(rows) for fr in range(pitch)}
    assert sorted(idx) == list(range(rows * pitch)), name
    # fragment view: every register's write (and read back) by the 32 lanes of a warp hits 32 distinct banks, and the warps
    # together cover every element of the slice exactly once
    seen = set()
    for w in range(4):
        for j, q in regs:
            cells = [frag(w, lane, j, q) for lane in range(32)]
            assert all(0 <= r < rows and 0 <= fr < pitch for r, fr in cells), (name, w, j, q)
            assert len({slot_index(r, fr, pitch) % 32 for r, fr in cells}) == 32, (name, w, j, q)
            seen.update(cells)
    assert len(seen) == rows * pitch, name
    # row view: warp w owns its rows whole; one instruction = frames l + 32 m of one row, 32 distinct banks
    assert sorted(r for wr in warp_rows for r in wr) == list(range(rows)), name
    for wr in warp_rows:
        for r in wr:
            for m in range(pitch // 32):
                assert len({slot_index(r, lane + 32 * m, pitch) % 32 for lane in range(32)}) == 32, (name, r, m)
