"""Host-side check of GEMM1's addressing in `block_fused_kernel` (fno_block_fused.cu), no GPU needed.

GEMM1's A fragments are read from the warpgroup's image slot, which its thread 0 fills by bulk copies of one ky pair of
the mode image, and its result goes to Zt, the K-major B operand of GEMM2, one 16-byte chunk per st.shared.v4.  A wrong offset in either would silently compute a different spectrum, so
both maps are replayed here for every thread of a CTA: each fragment register is loaded from the image byte that holds
the element (ky, kk, o) its GEMM1 row and K index stand for (the byte where the earlier kernel, with its producer warp
and its row order, read it), each accumulator value lands where GEMM2's descriptors read Zt[h'][o][2 ky + ri], and the
stores cover every word of a Zt row once.  The shared-memory wavefronts of each Zt store instruction are counted from
the bank of every word, and the slot's fill protocol is replayed for every CTA of batch sizes 1..600.  The offset
expressions are evaluated from the kernel source.
"""
import functools
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "cfdbench_b200", "csrc", "fno_block_fused.cu")
TC = os.path.join(ROOT, "cfdbench_b200", "csrc", "tc_common.cuh")

C, KX_ROWS, N_KY, ROWS = 32, 48, 12, 16   # channels, image rows (kx, re|im), ky modes, image rows per unit
KY_BYTES = KX_ROWS * C * 4                # 6144: one ky of the hi or the lo image
IMG_BYTES = 2 * N_KY * KY_BYTES           # 147456: one sample, hi then lo
ZT_FLOATS = C * 2 * N_KY                  # one Zt row, hi or lo: [32 o][24 k]


def _src():
    s = open(SRC).read()
    assert "constexpr size_t kYmImgBytes = %d;" % IMG_BYTES in s
    assert "constexpr uint32_t kImgKyBytes = kImgK * kC * 4;" in s
    assert "constexpr int kFzRows = %d;" % ROWS in s
    assert "constexpr int kFzThreads = 8 * 32;" in s
    # y_fill: the slot holds ky pair p = g + 2 (f % 3) of the unit's sample, hi at 0 and lo at kFzStage / 2
    assert "constexpr uint32_t kFzStage = 4 * kImgKyBytes;" in s
    assert ("img + static_cast<size_t>(b0 + (f / 3) * bstride) * kYmImgBytes +\n"
            "                               (g + 2 * (f % 3)) * (kFzStage / 2);") in s
    assert "bulk_g2s(sm.y[g], src, kFzStage / 2, &sm.y_full[g]);" in s
    assert "bulk_g2s(sm.y[g] + kFzStage / 2, src + kYmImgBytes / 2, kFzStage / 2, &sm.y_full[g]);" in s
    assert "mbar_expect_tx(&sm.y_full[g], kFzStage);" in s
    # load_pair: fragments from the slot
    assert "a[0][ks][r] = *reinterpret_cast<const uint32_t*>(sm.y[g] + off);" in s
    assert "a[1][ks][r] = *reinterpret_cast<const uint32_t*>(sm.y[g] + kFzStage / 2 + off);" in s
    # fills 3 u, 3 u + 1, 3 u + 2 go to a0, a1, a2, which GEMM1 issues as pairs g, g + 2, g + 4
    assert "first_pair(a0, 0);" in s and "first_pair(a1, 1);" in s and "first_pair(a2, 2);" in s
    assert "if (more && r == 1) load_pair(a0, 3 * u + 3);" in s
    assert "if (more && r == 3) load_pair(a1, 3 * u + 4);" in s
    assert "if (more && r == 5) load_pair(a2, 3 * u + 5);" in s
    assert "issue_pair(acc1[0], a0);" in s and "issue_pair(acc1[1], a1);" in s and "issue_pair(acc1[0], a2);" in s
    # store_pair: v[j] = acc[4 i + j], one float4 per hi / lo at (row 4 i + q, o1, k = 4 p)
    assert "float v[4] = {acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]};" in s
    assert "*reinterpret_cast<float4*>(&sm.zt[4 * i + q][0][off]) = hi;" in s
    assert "*reinterpret_cast<float4*>(&sm.zt[4 * i + q][1][off]) = lo;" in s
    assert "alignas(128) float zt[kFzRows][2][kFzZtFloats];" in s
    # GEMM2's B operand: row h', hi or lo, K step ks at + 2 ks LBO, SBO 128 (no swizzle)
    assert "tc::make_smem_desc(b_z[pass] + ks * 2 * kLboO, kLboO, 128)" in s
    assert "constexpr uint32_t kLboO = (kC / 8) * 128;" in s
    # GEMM1's three ky pairs per warpgroup g
    assert "store_pair(acc1[0], g);" in s and "store_pair(acc1[1], g + 2);" in s and "store_pair(acc1[0], g + 4);" in s

    def expr(pattern):
        m = re.search(pattern, s)
        assert m, pattern
        return m.group(1)

    return dict(
        o1=expr(r"const int o1 = ([^;]+);"),
        kk=expr(r"const int kk = ([^;]+);"),
        load_off=expr(r"const uint32_t off = (\(r & 1\) \* kImgKyBytes[^;]+);"),
        store_off=expr(r"const uint32_t off = (tc::kmajor_offset\(o1, [^;]+);"),
        lbo=(C // 8) * 128,
    )


@functools.lru_cache(None)
def _kmajor_fn():
    s = open(TC).read()
    m = re.search(r"kmajor_offset\(int row, int k, int rows\) \{\s*return static_cast<uint32_t>\((.+)\);\s*\}", s)
    assert m
    body = compile(m.group(1), TC, "eval")
    return lambda row, k, rows: eval(body, {}, dict(row=row, k=k, rows=rows))


_CODE = {}


def _ev(e, **v):
    if e not in _CODE:
        # C integer division on non-negative ints
        _CODE[e] = compile(e.replace("tc::kmajor_offset", "kmajor_offset").replace(" / ", " // "), SRC, "eval")
    return eval(_CODE[e], {"kmajor_offset": _kmajor_fn()}, v)


def _image_offset(hl, ky, kk, o):
    """byte of element (hi|lo, ky, line kk, channel o) in the mode image mode_mix_tc_kernel writes: [hl][ky][kk][32 o],
    32-byte chunk (o / 8) ^ (kk & 3) of the 128-byte line (tests/test_gpu_fused.py::encode_ym_image)"""
    return ((hl * N_KY + ky) * KX_ROWS + kk) * 128 + ((((o >> 3) ^ (kk & 3)) * 8) + (o & 7)) * 4


_IMAGE = {_image_offset(hl, ky, kk, o): (hl, ky, kk, o)
          for hl in range(2) for ky in range(N_KY) for kk in range(KX_ROWS) for o in range(C)}


def _staged_offset(hl, p, ky, kk, o):
    """where the earlier kernel read the same element: its stage held pair p (hi 12 KB, then lo) by two bulk copies from
    image bytes p * 12288 (hi) and 73728 + p * 12288 (lo); its GEMM1 row was m = (ky - 2p) * 32 + o"""
    m = (ky - 2 * p) * 32 + o
    off = (m >> 5) * 6144 + kk * 128 + (((o >> 3) ^ (kk & 3)) << 5) + (o & 7) * 4
    return hl * (IMG_BYTES // 2) + p * 2 * KY_BYTES + off


def _threads():
    for tid in range(256):
        warp, lane = tid // 32, tid % 32
        yield warp >> 2, warp & 3, lane, lane & 3


def _gemm1_rows(c):
    """for every thread and ky pair: the (ky, o) of fragment rows m0 (hh = 0) and m0 + 8 (hh = 1), from the loads"""
    rows = {}
    seen = np.zeros((2, N_KY, KX_ROWS, C), np.int32)
    for g, wq, lane, q in _threads():
        for p in (g, g + 2, g + 4):
            base = 2 * p * KY_BYTES
            for hh in range(2):
                elems = set()
                for ks in range(KX_ROWS // 8):
                    for r in (hh, hh + 2):
                        kk = _ev(c["kk"], ks=ks, q=q, r=r)
                        assert kk == 8 * ks + q + 4 * (r >> 1)   # the tf32 A fragment's K index of register r
                        off = _ev(c["load_off"], r=r, kk=kk, wq=wq, lane=lane, kImgKyBytes=KY_BYTES)
                        for hl in range(2):
                            got = base + hl * (IMG_BYTES // 2) + off
                            ghl, ky, gkk, o = _IMAGE[got]
                            assert (ghl, gkk) == (hl, kk) and ky in (2 * p, 2 * p + 1), (g, wq, lane, p, ks, r, hl)
                            assert got == _staged_offset(hl, p, ky, kk, o)
                            seen[hl, ky, kk, o] += 1
                            elems.add((ky, o))
                assert len(elems) == 1, "a fragment row mixes image rows"
                rows[(g, wq, lane, p, hh)] = elems.pop()
    return rows, seen


def test_fragment_loads_read_the_image_element_of_their_row():
    c = _src()
    rows, seen = _gemm1_rows(c)
    # one CTA loads every hi and lo element of the sample exactly once per unit
    assert np.all(seen == 1)
    # a GEMM1 tile of a ky pair holds all 64 (ky, o) rows, once each, per warpgroup
    for g in range(2):
        for p in (g, g + 2, g + 4):
            tile = [rows[(g, wq, lane, p, hh)] for wq in range(4) for lane in range(0, 32, 4) for hh in range(2)]
            assert sorted(tile) == [(ky, o) for ky in (2 * p, 2 * p + 1) for o in range(C)]
    # the thread's two rows are the pair's two ky at one channel, o1 = 8 wq + lane / 4
    for (g, wq, lane, p, hh), (ky, o) in rows.items():
        assert ky == 2 * p + hh and o == _ev(c["o1"], wq=wq, lane=lane)


def _zt_stores(c):
    """per store instruction (warp, ky pair, i, hl): per lane the 16-byte chunk it writes and the four (o, k) it holds"""
    rows, _ = _gemm1_rows(c)
    out = {}
    for g, wq, lane, q in _threads():
        warp = 4 * g + wq
        o1 = _ev(c["o1"], wq=wq, lane=lane)
        for p in (g, g + 2, g + 4):
            off = _ev(c["store_off"], o1=o1, p=p, kC=C)
            for i in range(4):
                hrow = 4 * i + q
                for hl in range(2):
                    byte = (hrow * 2 + hl) * ZT_FLOATS * 4 + off * 4
                    vals = []
                    for j in range(4):   # v[j] = acc[4 i + j] = D[m0 + 8 hh][8 i + 2 q + e], j = 2 hh + e
                        hh, e = j >> 1, j & 1
                        ky, o = rows[(g, wq, lane, p, hh)]
                        vals.append((hrow, hl, o, 2 * ky + e, byte + 4 * j))
                    out.setdefault((warp, p, i, hl), []).append((byte, 16, vals))
    return out


def _gemm2_read_offset(lbo, hrow, hl, o, k):
    """byte GEMM2's K-major B descriptor reads for Zt_h'[n = o][k]: start of (row, hl) + 2 ks LBO, then core matrix
    (k / 4 within the step) LBO apart along K and (o / 8) SBO = 128 apart along N, (o % 8) * 16 + (k % 4) * 4 inside"""
    ks, kin = divmod(k, 8)
    return (hrow * 2 + hl) * ZT_FLOATS * 4 + ks * 2 * lbo + (kin >> 2) * lbo + (o >> 3) * 128 + (o & 7) * 16 + (k & 3) * 4


def test_zt_stores_match_gemm2_descriptors():
    c = _src()
    words = {}
    for insts in _zt_stores(c).values():
        for byte, width, vals in insts:
            assert byte % width == 0
            for hrow, hl, o, k, b in vals:
                assert b == _gemm2_read_offset(c["lbo"], hrow, hl, o, k), (hrow, hl, o, k)
                assert b not in words, "two values stored to one word"
                words[b] = (hrow, hl, o, k)
    # a bijection onto each Zt row: every (o, k) of every (h', hi|lo) written exactly once
    assert sorted(words.values()) == [(h, hl, o, k) for h in range(ROWS) for hl in range(2) for o in range(C)
                                      for k in range(2 * N_KY)]


def _wavefronts(accesses):
    """shared-memory wavefronts of one warp-wide access: each wavefront serves one 4-byte word per bank and at most
    128 bytes, so the count is the larger of the most distinct words any bank holds and the bytes over 128"""
    per_bank = {}
    total = 0
    for byte, width in accesses:
        total += width
        for w in range(byte // 4, (byte + width) // 4):
            per_bank.setdefault(w % 32, set()).add(w)
    return max(max(len(v) for v in per_bank.values()), -(-total // 128)), total


def _old_scalar_stores():
    """the earlier kernel's Zt stores: one float per instruction (i, hh, e, hl), row m = (ky - 2p) * 32 + o of its tile"""
    out = {}
    for g, wq, lane, q in _threads():
        m0 = 16 * wq + (lane >> 2)
        for p in (g, g + 2, g + 4):
            for hh in range(2):
                m = m0 + 8 * hh
                ky, o = 2 * p + (m >> 5), m & 31
                for i in range(4):
                    for e in range(2):
                        k = 2 * ky + e
                        for hl in range(2):
                            byte = ((4 * i + q) * 2 + hl) * ZT_FLOATS * 4 + (((k >> 2) * 4 + (o >> 3)) * 128
                                                                              + (o & 7) * 16 + (k & 3) * 4)
                            out.setdefault((4 * g + wq, p, hh, i, e, hl), []).append((byte, 4))
    return out


def test_zt_store_wavefronts():
    c = _src()
    new = [_wavefronts([(b, w) for b, w, _ in insts]) for insts in _zt_stores(c).values()]
    assert all(wf * 128 <= 2 * nbytes for wf, nbytes in new)   # at most 2 wavefronts per 128 bytes stored
    assert {(wf, nbytes) for wf, nbytes in new} == {(4, 512)}  # 8 lanes per Zt row, 4 rows: one per 128 bytes
    old = [_wavefronts(a) for a in _old_scalar_stores().values()]
    assert {(wf, nbytes) for wf, nbytes in old} == {(4, 128)}  # four lanes of a quad, rows 6144 B apart: one bank
    assert len(new) * 4 == len(old)                           # 16-byte stores: a quarter of the instructions


def _slot_events(n_units, wg_rows=8):
    """program order of one warpgroup's image slot, as the kernel runs it: ('issue', f) by thread 0, ('wait', f) and
    ('read', f) by all threads, ('barrier',) = the 128-thread barrier after which thread 0 issues the next fill"""
    n = 3 * n_units
    ev = [("issue", 0)] if n > 0 else []
    if n_units > 0:
        for f in range(3):   # first_pair
            ev += [("wait", f), ("read", f), ("barrier",)]
            if f + 1 < n:
                ev.append(("issue", f + 1))
    for u in range(n_units):
        more = u + 1 < n_units
        for r in range(wg_rows + 1):
            if r < wg_rows and more and r in (1, 3, 5):
                f = 3 * u + 3 + r // 2
                ev += [("wait", f), ("read", f)]
            if r == 0:
                continue
            ev.append(("barrier",))
            if more and r in (1, 3, 5) and 3 * u + 4 + (r >> 1) < n:
                ev.append(("issue", 3 * u + 4 + (r >> 1)))
    return ev, n


def test_image_slot_protocol_all_batches():
    s = open(SRC).read()
    assert "if (t == 0 && f + 1 < n_yfills) y_fill(f + 1);" in s
    assert "if (more && (r == 1 || r == 3 || r == 5) && 3 * u + 4 + (r >> 1) < n_yfills) y_fill(3 * u + 4 + (r >> 1));" in s
    assert "const int n_yfills = 3 * n_units;" in s and "mbar_wait(&sm.y_full[g], f & 1);" in s
    seen = set()
    for n_sm in (132, 114):
        for batch in range(1, 601):
            slots = min(batch, n_sm // 4)
            for b0 in range(slots):
                seen.add((batch - b0 + slots - 1) // slots)
    for n_units in sorted(seen):
        ev, n = _slot_events(n_units)
        in_flight, landed, read, completed = None, None, [], 0
        unread_since_barrier = False
        for e in ev:
            if e[0] == "issue":
                f = e[1]
                # one fill in flight at a time, issued only after every thread read the previous one and met the barrier
                assert in_flight is None and landed is None and not unread_since_barrier, (n_units, f)
                assert f == (read[-1] + 1 if read else 0)
                in_flight = f
            elif e[0] == "wait":
                f = e[1]
                assert in_flight == f, (n_units, f)   # the wait can only pass once this fill has landed
                completed += 1
                assert completed - 1 == f and (completed - 1) & 1 == f & 1   # the phase its parity names
                landed, in_flight = f, None
            elif e[0] == "read":
                assert landed == e[1]
                read.append(e[1])
                landed, unread_since_barrier = None, True
            else:
                unread_since_barrier = False
        assert read == list(range(n)) and in_flight is None   # every fill read once, nothing in flight at exit
