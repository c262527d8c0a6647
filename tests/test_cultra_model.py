"""The ULTRA model (tests/cultra.py) on the CPU: its far walk is a brute-force search; where the window is 131072 it is OPT; each of
its rules holds on a crafted input; its frames decode through libzstd and the oracle at window_log 18, 20, 23 and 27; and on 4 MiB
of text at window_log 22 its ratio is above OPT's and libzstd level 3's."""
import hashlib
import random

import pytest

import cldm
import clazy
import copt
import cparse
import cultra
import datagen
import test_gpu_cultra

B, W = cparse.BLOCK, cparse.WINDOW


def rand(seed, n):
    return bytearray(random.Random(seed).randbytes(n))


def offsets(blocks):
    return cldm.offsets(blocks)


def sequences(blocks):
    """(block, position in the block, ml, of) of every sequence of a frame's parse."""
    out = []
    for k, b in enumerate(blocks):
        if b[0] == "rle":
            continue
        pos = 0
        for ll, ml, of in b[1]:
            pos += ll
            out.append((k, pos, ml, of))
            pos += ml
    return out


def test_far_walk_is_the_brute_force_search():
    buf = rand(1, 700000)
    pat = bytes(rand(2, 8))
    rng = random.Random(3)
    for _ in range(400):                            # one key at many places, some 8-byte copies of earlier bytes
        at = rng.randrange(0, len(buf) - 8)
        buf[at:at + 8] = pat if rng.random() < 0.5 else buf[at // 2:at // 2 + 8]
    F = bytes(buf)
    for wf in (1 << 18, 1 << 19, 1 << 20):
        ff = cultra.FarFrame(F, wf)
        qs = [q for q in range(W + 1, len(F), 997)] + [q for q in range(len(F)) if F[q:q + 8] == pat][:200]
        for q in qs:
            assert ff.walk(q) == cultra.brute_far(F, q, wf), (wf, q)
    keyed = cultra.keys(F) >= 0
    assert not keyed[B - 7:B].any() and keyed[B - 8] and keyed[B] and not keyed[len(F) - 7:].any()


def test_ultra_is_opt_where_the_window_is_131072():
    small = [c.frames for c in copt.cases() if c.content is None and all(len(f) <= B for f in c.frames)][:12]
    for frames in small:
        assert cparse.parse(frames, None, cultra.level(27)) == cparse.parse(frames, None, copt.OPT)
    big = test_gpu_cultra.inputs()[0][:600000]
    assert cultra.parse([big], 17) == cldm.parse([big], 17, None, copt.OPT)


def far_frame(n, dst, src, ln, seed=5):
    buf = rand(seed, n)
    buf[dst:dst + ln] = buf[src:src + ln]
    return bytes(buf)


@pytest.mark.parametrize("o,found", [(W + 1, True), (1 << 18, True), ((1 << 18) + 1, False)], ids=["131073", "Wf", "Wf+1"])
def test_far_match_reach(o, found):
    """A 24-byte copy o bytes back in a 300,000-byte frame at window_log 18 (Wf = 2^18)."""
    dst = 290000 - 24
    F = far_frame(300000, dst, dst - o, 24)
    seqs = sequences(cultra.parse([F], 18)[0])
    assert ((2, dst - 2 * B, 24, o) in seqs) == found
    assert all(of <= 1 << 18 for _, _, _, of in seqs)


def test_depth_cap_counts_every_entry():
    """One 8-byte pattern at FAR_DEPTH + 1 places far back; only the farthest continues as q does: the walk stops before it."""
    n = 700000
    buf = rand(6, n)
    pat = bytes(rand(7, 8))
    q = 650000
    for k in range(cultra.FAR_DEPTH + 1):
        at = q - W - 1000 - 3000 * k
        buf[at:at + 8] = pat
    far_at = q - W - 1000 - 3000 * cultra.FAR_DEPTH
    buf[q:q + 8] = pat
    buf[far_at + 8:far_at + 40] = buf[q + 8:q + 40]
    F = bytes(buf)
    ff = cultra.FarFrame(F, 1 << 20)
    walk = ff.walk(q)
    assert len(walk) == cultra.FAR_DEPTH and far_at not in walk
    cultra.FAR_DEPTH += 1
    try:
        assert far_at in cultra.FarFrame(F, 1 << 20).walk(q)
    finally:
        cultra.FAR_DEPTH -= 1


def test_near_beats_far_of_equal_length():
    n = 400000
    buf = rand(8, n)
    q = 350000
    buf[q - 1000:q - 1000 + 12] = buf[q:q + 12]
    buf[q - 200000:q - 200000 + 12] = buf[q:q + 12]
    F = bytes(buf)
    far = cultra.Far(20)
    ff = far.frame(F)
    base = (q // B) * B
    prev = copt.chain(cparse.hashes(F, copt.OPT_HASH_LOG))
    got = ff.candidates(F, base, base, q - base, B, prev, None, None)
    assert [(ln, o) for ln, o, _ in got] == [(12, 1000)]
    assert q - 200000 in ff.walk(q)


def test_repeat_of_a_far_offset_and_of_a_forced_piece():
    n = 900000
    buf = rand(9, n)
    o = 300000
    buf[600000:600000 + 20] = buf[600000 - o:600000 - o + 20]          # a far match
    buf[600040:600040 + 9] = buf[600040 - o:600040 - o + 9]            # then its offset again, as a repeat
    p = 200000
    buf[700000:700000 + 4000] = buf[700000 - p:700000 - p + 4000]       # a forced piece (>= 64 bytes, around an anchor)
    buf[704030:704030 + 9] = buf[704030 - p:704030 - p + 9]            # then its offset as a repeat
    F = bytes(buf)
    blocks = cultra.parse([F], 20)[0]
    seqs = sequences(blocks)
    at = {(k * B + pos, of) for k, pos, _, of in seqs}
    assert (600000, o) in at and (600040, o) in at
    assert (704030, p) in at
    assert cldm.forced([F], 20)[0][700000 // B]
    recs = {}
    for k, b in enumerate(blocks):
        pos = 0
        for (ll, ml, of), r in zip(b[1], clazy.records(b[1])):
            pos += ll
            recs[k * B + pos] = r[2]
            pos += ml
    assert all((recs[x] + 3) % (1 << 32) <= 3 for x in (600040, 704030))   # coded as repeats (Offset_Value 1..3)


def test_matches_stop_at_the_segment_end():
    n = 3 * B
    buf = rand(10, n)
    seglen = B // cparse.CM_WARPS
    for w in range(1, cparse.CM_WARPS):
        s = 2 * B + w * seglen
        buf[s - 16:s + 48] = buf[s - 16 - 200000:s + 48 - 200000]
    F = bytes(buf)
    for k, pos, ml, of in sequences(cultra.parse([F], 20)[0]):
        if k == 2:
            assert pos // seglen == (pos + ml - 1) // seglen
    assert any(of == 200000 for *_, of in sequences(cultra.parse([F], 20)[0]))


@pytest.mark.parametrize("window_log", [18, 20, 23, 27])
def test_round_trips(oracle, window_log):
    data = test_gpu_cultra.inputs()[0]
    blocks = cultra.parse([data], window_log)[0]
    f = cultra.reference_frame(data, blocks, window_log)
    assert any(o > W for o in offsets(blocks))
    assert datagen.decompress(f, len(data), window_log_max=27) == data
    o = oracle.FrameDecoder()
    o.set_max_window_size(1 << 27)
    o.decode_blocks(o.reset(f))
    assert o.collect() == data


def test_ratio_above_opt_and_libzstd_level3_at_window_log_22():
    data = bytes(datagen.gen_text(4 << 20, 0xE90001))
    f = cultra.reference_frame(data, cultra.parse([data], 22)[0], 22)
    o = cparse.reference_frame(data, cldm.parse([data], 22, None, copt.OPT)[0], level=copt.OPT, window_log=22)
    z3 = len(datagen.compress(data, level=3, window_log=22))
    print(f"ULTRA model {len(data) / len(f):.4f}, OPT model {len(data) / len(o):.4f}, libzstd level 3 {len(data) / z3:.4f}")
    assert len(f) < len(o) and len(f) < z3
    assert (len(f), hashlib.sha256(f).hexdigest()) == (test_gpu_cultra.RATIO_FRAME_LEN, test_gpu_cultra.RATIO_FRAME_SHA)
