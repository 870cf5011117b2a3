"""Host-side check of the activation-ring protocol of `block_fused_kernel` (fno_block_fused.cu), no GPU needed.

The kernel's warpgroup g walks GEMM2 rows as one fill counter n = 8 u + r over its units; fill n lands in slot n % S and
completes phase n / S of that slot's mbarrier; its thread 0 issues the first S fills up front and fill n + S right after
the barrier that follows row n's epilogue.  A wrong slot, parity or byte count would stall a wait until the bounded spin
traps, so the arithmetic is replayed here for every CTA of every batch size 1..600 on 132- and 114-SM parts: program
order of issues and waits, the mbarrier phase each wait observes, the TMA coordinates against the map, and that every
activation row is loaded and every output row stored exactly once.  The constants are read from the kernel source.
"""
import os
import re

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfdbench_b200", "csrc",
                   "fno_block_fused.cu")


def _consts():
    s = open(SRC).read()

    def get(name):
        m = re.search(r"constexpr\s+(?:int|uint32_t)\s+[^;]*\b" + name + r"\s*=\s*(\d+)\s*[,;]", s)
        assert m, name
        return int(m.group(1))

    assert "kFzRows = 16;" in s and "kFzWgRows = kFzRows / 2;" in s and "kFzChunks = kH / kFzRows;" in s
    assert "return n % kFzXSlots;" in s and "(n / kFzXSlots) & 1u" in s
    assert "kFzRowBytes = kFzBoxW * kFzBoxH * kFzBoxC * 2;" in s
    assert "mbar_expect_tx(&sm.x_full[g][s], kFzRowBytes);" in s
    assert "mbar_init(&sm.x_full[i][s], 1);" in s
    assert "kFzBoxW = kW, kFzBoxH = 1, kFzBoxC = kC;" in s
    return dict(S=get("kFzXSlots"), rows=16, wg_rows=8, chunks=4)


def _ring_events(n_units, S, wg_rows):
    """program order of thread 0 / the warpgroup for one ring: ('issue', n) and ('wait', n), as the kernel runs them"""
    n_fills = wg_rows * n_units
    ev = [("issue", n) for n in range(min(S, n_fills))]
    for u in range(n_units):
        for r in range(wg_rows + 1):
            if r < wg_rows:
                ev.append(("wait", wg_rows * u + r))
            if r == 0:
                continue
            nf = wg_rows * u + (r - 1) + S
            ev.append(("release", wg_rows * u + r - 1))
            if nf < n_fills:
                ev.append(("issue", nf))
    return ev, n_fills


def _check_ring(n_units, S, wg_rows):
    ev, n_fills = _ring_events(n_units, S, wg_rows)
    completed = [0] * S        # phases completed per slot (a fill completes once its bytes land)
    armed = [None] * S         # fill currently in flight in the slot
    released = set()
    waited = []
    for kind, n in ev:
        s = n % S
        if kind == "issue":
            assert armed[s] is None, ("slot refilled while a fill is pending", n)
            assert n < S or (n - S) in released, ("slot refilled before its reader finished", n)
            armed[s] = n
        elif kind == "wait":
            # the earliest the wait can pass: the fill it waits for has landed
            assert armed[s] == n, ("waiting for a fill that was never issued", n)
            completed[s] += 1
            armed[s] = None
            phase = completed[s] - 1
            assert phase == n // S and (phase & 1) == ((n // S) & 1), ("parity", n)
            waited.append(n)
        else:
            assert n in waited
            released.add(n)
    assert waited == list(range(n_fills))
    assert all(a is None for a in armed)   # nothing in flight at exit


def test_ring_protocol_all_batches():
    c = _consts()
    S, wg_rows, chunks = c["S"], c["wg_rows"], c["chunks"]
    assert 2 <= S <= 8
    seen = set()
    for n_sm in (132, 114):
        for batch in range(1, 601):
            slots = min(batch, n_sm // chunks)
            for b0 in range(slots):
                seen.add((batch - b0 + slots - 1) // slots)
    for n_units in sorted(seen):
        _check_ring(n_units, S, wg_rows)


def test_tma_boxes_cover_each_row_once():
    c = _consts()
    rows, wg_rows, chunks = c["rows"], c["wg_rows"], c["chunks"]
    for n_sm in (132, 114):
        for batch in range(1, 601):
            slots = min(batch, n_sm // chunks)
            hits = np.zeros((batch, 64), np.int32)
            for cta in range(chunks * slots):
                chunk, b0, bstride = cta % chunks, cta // chunks, slots
                n_units = (batch - b0 + bstride - 1) // bstride if b0 < batch else 0
                for g in range(2):
                    for n in range(wg_rows * n_units):
                        u, r = divmod(n, wg_rows)
                        h, plane0 = rows * chunk + g + 2 * r, (b0 + u * bstride) * 32
                        # box {64, 1, 32} at {0, h, plane0} inside dims {64, 64, 32 batch}
                        assert 0 <= h < 64 and 0 <= plane0 and plane0 + 32 <= 32 * batch
                        hits[plane0 // 32, h] += 1
            assert np.all(hits == 1), (n_sm, batch)


def test_tensor_map_parameters():
    """cuTensorMapEncodeTiled limits for the x / out maps at the batch sizes the GPU tests use"""
    elt = 2
    for batch in (1, 3, 80, 256, 1000):
        dims = (64, 64, 32 * batch)
        strides = (64 * elt, 64 * 64 * elt)
        box = (64, 1, 32)
        assert all(1 <= d <= 2 ** 32 for d in dims)
        assert all(s % 16 == 0 and s < 2 ** 40 for s in strides)
        assert all(1 <= b <= 256 and b <= d for b, d in zip(box, dims))
        assert box[0] * elt <= 128            # 128-byte swizzle: the inner box extent is one 128-byte line
        assert box[0] * box[1] * box[2] * elt == 4096
