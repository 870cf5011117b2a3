"""Host-side check of the unit mapping, TMA ring and shared-memory swizzle of `dft_fwd_tc_kernel` (fno_dft_fwd_tc.cu),
no GPU needed.

A unit is eight planes of one sample.  Warpgroup pipeline `first` of the grid takes units first, first + stride, ...;
its fill n is box n % 4 (two planes, 16 KB) of its unit n / 4, lands in slot n % S and completes phase n / S of that
slot's mbarrier; thread 0 issues the first S fills up front and fill n + S once stage A has read fill n.  A wrong slot,
parity or coordinate would stall a wait until the bounded spin traps or read the wrong planes, so the arithmetic is
replayed here for every CTA of every batch size 1..600 on 132- and 114-SM parts: program order of issues and waits, the
phase each wait observes, the box coordinates against the tensor map, and that every plane is loaded and every
spectrum element written exactly once.  The functions are restated from the kernel source, which is checked to still
contain them.
"""
import os
import re

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfdbench_b200", "csrc",
                   "fno_dft_fwd_tc.cu")


def _src():
    return open(SRC).read()


def _consts():
    s = _src()

    def get(name):
        m = re.search(r"constexpr\s+(?:int|uint32_t)\s+" + name + r"\s*=\s*(\d+)\s*;", s)
        assert m, name
        return int(m.group(1))

    for line in ("return n % kTdSlots;",
                 "return static_cast<uint32_t>(n / kTdSlots) & 1u;",
                 "return (unit * kTdPlanes + box * kTdBoxPlanes) * kH;",
                 "return first + i * stride;",
                 "return first < n_units ? (n_units - first + stride - 1) / stride : 0;",
                 "return m * kTdK2 + (h ^ (((m & 7) << 2) ^ (((m >> 4) & 3) << 3)));",
                 "mbar_expect_tx(bar, kTdBoxBytes);",
                 "td_box_row(td_unit(first, stride, n / kTdBoxes), n % kTdBoxes)",
                 "mbar_init(&sm.x_full[i][s], 1);",
                 "const int first = blockIdx.x * kTdWG + wg, stride = gridDim.x * kTdWG;",
                 "const int n_units = batch * kC / kTdPlanes;",
                 "kTdBoxPlanes * kH);",
                 "const int b = unit * kTdPlanes / kC, c0 = unit * kTdPlanes % kC;",
                 "xm[(static_cast<size_t>(kxi * kM2 + qq) * batch + b) * kC + c0 + lr]"):
        assert line in s, line
    assert "constexpr int kTdBoxes = kTdPlanes / kTdBoxPlanes;" in s
    assert "constexpr uint32_t kTdBoxBytes = kTdBoxPlanes * kTdPlaneBytes;" in s
    return dict(S=get("kTdSlots"), planes=get("kTdPlanes"), box_planes=get("kTdBoxPlanes"), wg=get("kTdWG"))


def _grid(batch, n_sm, c):
    n_units = batch * 32 // c["planes"]
    per_pipe = -(-n_units // (c["wg"] * n_sm))
    return n_units, -(-n_units // (c["wg"] * per_pipe))


def _units_of(first, stride, n_units):
    return (n_units - first + stride - 1) // stride if first < n_units else 0


def _check_ring(n_fills, S):
    """program order of one pipeline: thread 0 issues fills 0..S-1, the warpgroup waits for fill n, stage A reads it,
    then thread 0 issues fill n + S"""
    armed = [None] * S          # fill in flight per slot
    completed = [0] * S         # phases completed per slot
    for n in range(min(S, n_fills)):
        assert armed[n % S] is None
        armed[n % S] = n
    for n in range(n_fills):
        s = n % S
        assert armed[s] == n, ("waiting for a fill that was never issued", n)
        armed[s] = None
        completed[s] += 1
        phase = completed[s] - 1
        assert phase == n // S and (phase & 1) == ((n // S) & 1), ("parity", n)
        if n + S < n_fills:
            assert armed[(n + S) % S] is None, ("slot refilled while a fill is pending", n + S)
            armed[(n + S) % S] = n + S
    assert all(a is None for a in armed)


def test_ring_protocol_all_batches():
    c = _consts()
    S, boxes = c["S"], c["planes"] // c["box_planes"]
    assert 2 <= S <= 8 and boxes * c["box_planes"] == c["planes"]
    seen = set()
    for n_sm in (132, 114):
        for batch in range(1, 601):
            n_units, grid = _grid(batch, n_sm, c)
            stride = grid * c["wg"]
            seen.update(_units_of(f, stride, n_units) for f in range(stride))
    for n in sorted(seen):
        _check_ring(n * boxes, S)


def test_units_cover_planes_and_spectrum_once():
    c = _consts()
    planes, box_planes, wg = c["planes"], c["box_planes"], c["wg"]
    boxes = planes // box_planes
    for n_sm in (132, 114):
        for batch in range(1, 601):
            n_units, grid = _grid(batch, n_sm, c)
            assert 1 <= grid <= n_sm
            stride = grid * wg
            counts = [_units_of(f, stride, n_units) for f in range(stride)]
            assert max(counts) == -(-n_units // (wg * n_sm)), (n_sm, batch)   # as short as a full grid
            loaded = np.zeros(batch * 32, np.int32)
            written = np.zeros(batch * 32, np.int32)    # per (sample, channel); each covers the 288 modes
            for first in range(stride):
                for i in range(counts[first]):
                    unit = first + i * stride
                    for k in range(boxes):
                        row = (unit * planes + k * box_planes) * 64
                        assert row % 64 == 0 and 0 <= row and row + box_planes * 64 <= batch * 32 * 64
                        loaded[row // 64:row // 64 + box_planes] += 1
                    b, c0 = unit * planes // 32, unit * planes % 32
                    assert b < batch and c0 + planes <= 32
                    written[b * 32 + c0:b * 32 + c0 + planes] += 1
            assert np.all(loaded == 1) and np.all(written == 1), (n_sm, batch)


def _g_index(m, h):
    return m * 64 + (h ^ (((m & 7) << 2) ^ (((m >> 4) & 3) << 3)))


def test_g_buffer_swizzle_is_conflict_free():
    """the G buffer [192][64] fp32: a permutation of each row; the stage-A stores (lane = (h % 8, q % 4)) and the
    stage-B A-fragment loads (lane = (plane, h % 4)) of one warp instruction hit 32 distinct banks"""
    for m in range(192):
        assert sorted(_g_index(m, h) for h in range(64)) == list(range(64 * m, 64 * m + 64))
    for wq in range(4):
        for g3 in range(3):
            for hh in range(2):
                for ri in range(2):
                    for plane in range(8):
                        banks = {_g_index(16 * (4 * g3 + lane % 4) + 8 * ri + plane, 16 * wq + lane // 4 + 8 * hh) % 32
                                 for lane in range(32)}
                        assert len(banks) == 32
        for tile in range(3):
            for ks in range(8):
                for r in range(4):
                    banks = {_g_index(64 * tile + 16 * wq + lane // 4 + 8 * (r & 1), 8 * ks + lane % 4 + 4 * (r >> 1)) % 32
                             for lane in range(32)}
                    assert len(banks) == 32

