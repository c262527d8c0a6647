"""The plain model of the LAZY level (tests/clazy.py) checked against the format, without the GPU: every case's parse replays to
its input within the window, the frame and the segment; the frames reference_frame assembles decode with the oracle and libzstd,
and the oracle's trace shows repeat codes; hand-computed parses and repeat-offset passes match; each crafted case hits the rule
it is named after; and on 64 frames of 128 KiB of C2b-shaped text the model's ratio is at least libzstd level 1's."""
import os

import pytest

import clazy
import cparse
import datagen
import seqcraft

pytestmark = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")
CASES = clazy.cases()
_parsed = {}


def parsed(c):
    if c.id not in _parsed:
        _parsed[c.id] = cparse.parse(c.frames, c.content, clazy.LAZY)
    return _parsed[c.id]


def by_id(name):
    return next(c for c in CASES if c.id == name)


def positions(seqs):
    """(position in the block, ml, offset) of every sequence."""
    p, out = 0, []
    for ll, ml, of in seqs:
        p += ll
        out.append((p, ml, of))
        p += ml
    return out


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_parse_obeys_the_format(c):
    tail = len(cparse.match_dict(c.content).data) if cparse.match_dict(c.content) else 0
    pre = [("raw", c.content)] if c.content else []
    for data, blocks in zip(c.frames, parsed(c)):
        cmp = [b if b[0] == "rle" else ("cmp", b[0], b[1]) for b in blocks]
        out = seqcraft.execute(pre + cmp)
        assert out is not seqcraft.ERROR and out[len(c.content or b""):] == data
        ov = [b if b[0] == "rle" else ("cmp", b[0], clazy.reps(b[1])) for b in blocks]   # the coded offsets replay too
        out = seqcraft.execute(pre + ov, ov=True)
        assert out is not seqcraft.ERROR and out[len(c.content or b""):] == data
        for k, b in enumerate(blocks):
            if b[0] == "rle":
                continue
            n = min(cparse.BLOCK, len(data) - k * cparse.BLOCK)
            seglen = -(-n // cparse.CM_WARPS)
            for pos, ml, of in positions(b[1]):
                fpos = k * cparse.BLOCK + pos
                assert ml >= clazy.MIN_MATCH and 1 <= of <= clazy.WINDOW
                assert pos // seglen == (pos + ml - 1) // seglen, "a match crosses its segment's end"
                if of > fpos:
                    assert k == 0 and of - fpos <= tail and ml <= of - fpos, "a dictionary source past the dictionary's end"


def traced(oracle, f, content=None):
    d = oracle.FrameDecoder()
    d.trace_enable()
    if content is not None:
        d.add_raw_content_dict(1, content)
    r = d.reset(f)
    if content is not None:
        d.force_dict(1)
    d.decode_blocks(r)
    d.collect()
    return d.trace()[2]


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_reference_frame_decodes(oracle, c):
    reps = 0
    for data, blocks in zip(c.frames, parsed(c)):
        f = cparse.reference_frame(data, blocks, level=clazy.LAZY)
        assert datagen.decompress(f, len(data), raw_dict=c.content) == data
        assert oracle.decode_frame(f, raw_dict=c.content)[0] == data
        seqs = traced(oracle, f, c.content)
        assert all(int(s[3]) <= clazy.WINDOW for s in seqs)
        reps += sum(1 for s in seqs if int(s[2]) <= 3)
    if c.group == "data":
        assert reps > 50, "the realistic cases code repeat offsets"


def test_hand_computed_parses():
    # 40 bytes: seglen 5; segment 1 repeats segment 0 (found through t1), its literals carry on
    d = bytes(range(0x20, 0x25)) * 2 + bytes(range(0x60, 0x7e))
    assert cparse.parse([d], level=clazy.LAZY) == [[(d[:5] + d[10:], [(5, 5, 5)])]]
    # 256 bytes: seglen 32; a 40-byte repeat inside segment 3 from segment 0 is verified to 32 = e - q and not extended
    d = bytearray(range(256))
    d[100:128] = d[4:32]
    d = bytes(d)
    assert cparse.parse([d], level=clazy.LAZY)[0][0][1] == [(100, 28, 96)]
    # a dictionary of 5 bytes; all equal, empty, too short
    d = b"hello" + bytes(range(0x60, 0x83))
    assert cparse.parse([d], b"hello", clazy.LAZY) == [[(d[5:], [(0, 5, 5)])]]
    assert cparse.parse([b"zzzz", b"", b"abcd"], level=clazy.LAZY) == [[("rle", ord("z"), 4)], [(b"", [])], [(b"abcd", [])]]


def test_hand_computed_repeat_codes():
    # LL > 0: rep0 / rep1 / rep2 -> 1 / 2 / 3 once known; unknown slots are never named
    assert clazy.reps([(1, 5, 100), (1, 5, 100), (1, 5, 200), (1, 5, 100), (1, 5, 300), (1, 5, 100)]) == \
        [(1, 5, 103), (1, 5, 1), (1, 5, 203), (1, 5, 2), (1, 5, 303), (1, 5, 2)]
    # LL = 0: rep1 -> 1, rep2 -> 2, rep0 - 1 -> 3; rep0 itself cannot be named, so it is coded raw
    assert clazy.reps([(1, 5, 100), (1, 5, 200), (0, 5, 100)]) == [(1, 5, 103), (1, 5, 203), (0, 5, 1)]
    assert clazy.reps([(1, 5, 100), (1, 5, 200), (1, 5, 300), (0, 5, 100)]) == [(1, 5, 103), (1, 5, 203), (1, 5, 303), (0, 5, 2)]
    assert clazy.reps([(1, 5, 100), (0, 5, 99)]) == [(1, 5, 103), (0, 5, 3)]
    assert clazy.reps([(1, 5, 100), (0, 5, 100)]) == [(1, 5, 103), (0, 5, 103)]
    assert clazy.reps([(0, 5, 7)]) == [(0, 5, 10)]                       # an unknown rep0 - 1 is never named
    assert clazy.records([(1, 5, 100), (1, 5, 100)]) == [(1, 5, 100), (1, 5, 0xFFFFFFFE)]


def seqs_at(c, block=-1):
    return positions(parsed(c)[0][block][1])


def test_cases_hit_their_rule():
    z = cparse.seg_bounds(40000, 1)[0] + 32 * 40 + 3
    assert (z + 1, 30, z + 1 - 1000) in seqs_at(by_id("lazy-later-lane-wins"))                       # lane z + 1 beats z
    z = cparse.seg_bounds(40000, 3)[0] + 32 * 40 + 3
    assert (z, 8, 5000) in seqs_at(by_id("lazy-tie-keeps-first-lane"))                                 # a tie keeps lane z
    c = by_id("rep-found-where-t1-and-table-miss")
    assert (70500, 20, 68000) in seqs_at(c)
    assert clazy.reps(parsed(c)[0][0][1])[-1][2] == 1
    c = by_id("rep-ll0-rep0-across-segment-start")
    s = cparse.seg_bounds(cparse.BLOCK, 3)[0]
    assert seqs_at(c)[-2:] == [(s - 32, 32, 268), (s, 32, 268)]
    assert [r[2] for r in clazy.reps(parsed(c)[0][0][1])][-2:] == [271, 271]                          # LL = 0, rep0: raw
    c = by_id("rep-block-starts-with-previous-blocks-offset")
    assert seqs_at(c, 0)[-1][2] == seqs_at(c, 1)[0][2] == 1000
    assert clazy.reps(parsed(c)[0][1][1])[0][2] == 1003                                                # the history starts unknown
    a, z = cparse.BLOCK - 1000, 3000
    assert (z, 20, z + 1000) in seqs_at(by_id("bucket-K-1-newer-keep"))
    assert (z + 1, 19, z + 1000) in seqs_at(by_id("bucket-K-newer-evict"))
    S = clazy.LZ_SEED
    assert seqs_at(by_id(f"seed-source-{S}-before-segment=LZ_SEED"))[0] == (2000, 24, S + 2000)
    assert seqs_at(by_id(f"seed-source-{S + 1}-before-segment=LZ_SEED+1"))[0] == (2001, 23, S + 2001)
    assert seqs_at(by_id("dict-rep-source-before-frame")) == [(100, 20, 2100), (160, 20, 660)]
    assert seqs_at(by_id("dict-in-frame-as-long-as-dict"))[1][2] == 19900
    assert seqs_at(by_id("dict-len4=MIN_MATCH-1")) == [] and seqs_at(by_id("dict-len5=MIN_MATCH"))[0] == (0, 5, 5)


def test_ratio_at_least_libzstd_level1():
    """64 frames of 128 KiB of C2b-shaped text: the model's frames against libzstd 1.5.5 level 1 with a 128 KiB window."""
    from concurrent.futures import ProcessPoolExecutor
    plain = datagen.c2_text_plain(64 * 131072).tobytes()
    datas = [plain[i:i + 131072] for i in range(0, len(plain), 131072)]
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:   # parse in parallel, encode here
        blocks = list(ex.map(cparse.parse_frame, datas, [clazy.LAZY] * len(datas)))
    ratio = len(plain) / sum(len(cparse.reference_frame(d, b, level=clazy.LAZY)) for d, b in zip(datas, blocks))
    zstd1 = len(plain) / sum(len(datagen.compress(d, level=1, window_log=17)) for d in datas)
    print(f"LAZY model ratio {ratio:.3f}, libzstd level 1 {zstd1:.3f}")
    assert ratio >= zstd1

