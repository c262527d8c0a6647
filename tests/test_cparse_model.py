"""The plain model of the compressor's parse (tests/cparse.py) checked against the format, without the GPU: every case's parse
replays to its input, keeps its offsets inside the window and the frame (or the dictionary), never runs a match past its segment's
end or a dictionary source past the dictionary's end, and accounts for every byte; the frames reference_frame assembles decode
with the oracle and libzstd; a few tiny inputs have hand-computed parses; the crafted cases hit the rule they are named after;
and the plain XXH64 gives the known answers."""
import os
import random

import pytest

import cparse
import datagen
import seqcraft

pytestmark = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")
CASES = cparse.cases()
_parsed = {}


def parsed(c):
    if c.id not in _parsed:
        _parsed[c.id] = cparse.parse(c.frames, c.content)
    return _parsed[c.id]


def replay(blocks, content=None):
    """The bytes the blocks decode to, a raw-content dictionary's content standing before the frame."""
    pre = [("raw", content)] if content else []
    cmp = [b if b[0] == "rle" else ("cmp", b[0], b[1]) for b in blocks]
    out = seqcraft.execute(pre + cmp)
    assert out is not seqcraft.ERROR
    return out[len(content or b""):]


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_parse_obeys_the_format(c):
    tail = len(cparse.match_dict(c.content).data) if cparse.match_dict(c.content) else 0
    for data, blocks in zip(c.frames, parsed(c)):
        assert replay(blocks, c.content) == data
        assert len(blocks) == max(1, -(-len(data) // cparse.BLOCK))
        for k, b in enumerate(blocks):
            n = min(cparse.BLOCK, len(data) - k * cparse.BLOCK)
            if b[0] == "rle":
                assert b[2] == n and data[k * cparse.BLOCK:k * cparse.BLOCK + n] == bytes([b[1]]) * n
                continue
            lits, seqs = b
            assert len(lits) + sum(ml for _, ml, _ in seqs) == n
            seglen = -(-n // cparse.CM_WARPS)
            pos = 0                                                 # in the block
            for ll, ml, of in seqs:
                pos += ll
                fpos = k * cparse.BLOCK + pos                       # in the frame
                assert ml >= cparse.MIN_MATCH and 1 <= of <= cparse.WINDOW
                assert pos // seglen == (pos + ml - 1) // seglen, "a match crosses its segment's end"
                if of > fpos:
                    assert k == 0 and of - fpos <= tail and ml <= of - fpos, "a dictionary source past the dictionary's end"
                pos += ml


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_reference_frame_decodes(oracle, c):
    for data, blocks in zip(c.frames, parsed(c)):
        f = cparse.reference_frame(data, blocks)
        assert datagen.decompress(f, len(data), raw_dict=c.content) == data
        assert oracle.decode_frame(f, raw_dict=c.content)[0] == data
        assert cparse.reference_frame(data, blocks, level=cparse.UNCOMPRESSED) == oracle_free_raw(data)


def oracle_free_raw(data):
    """The Uncompressed level's frame written out by hand: header, Raw blocks, checksum."""
    import struct
    out = cparse.frame_header(len(data), True)
    pieces = [data[i:i + cparse.BLOCK] for i in range(0, len(data), cparse.BLOCK)] or [b""]
    for k, p in enumerate(pieces):
        out += struct.pack("<I", (1 if k == len(pieces) - 1 else 0) | (len(p) << 3))[:3] + p
    return out + struct.pack("<I", cparse.xxh64(data) & 0xFFFFFFFF)


def unique(n, start=0x20):
    return bytes(range(start, start + n))


def test_hand_computed_parses():
    # 40 bytes: seglen 5, one valid lane per segment (q = s); segment 1 repeats segment 0, found through t1 at its first byte;
    # segment 0's literals carry into segment 1's sequence
    d = unique(5) + unique(5) + unique(30, 0x60)
    assert cparse.parse([d]) == [[(d[:5] + d[10:], [(5, 5, 5)])]]
    # 80 bytes: seglen 10; the repeat fills segment 1 (verified for min(16, e - q) = 10 bytes, so not extended)
    d = unique(10) + unique(10) + unique(60, 0x60)
    assert cparse.parse([d]) == [[(d[:10] + d[20:], [(10, 10, 10)])]]
    # 256 bytes: seglen 32; a 40-byte repeat inside segment 3 from segment 0: verified to CM_CAP, extended to the segment's end
    d = bytearray(range(256))
    d[100:128] = d[4:32]
    d = bytes(d)
    lits, seqs = cparse.parse([d])[0][0]
    assert seqs == [(100, 28, 96)] and lits == d[:100] + d[128:]
    # all equal, empty, too short to match
    assert cparse.parse([b"zzzz", b"", b"abcd"]) == [[("rle", ord("z"), 4)], [(b"", [])], [(b"abcd", [])]]
    # a 5-byte dictionary: position 0 matches its only position at offset 0 + 5 - 0
    d = b"hello" + unique(35, 0x60)
    assert cparse.parse([d], b"hello") == [[(d[5:], [(0, 5, 5)])]]
    assert cparse.parse([d], b"hell") == [[(d, [])]]          # shorter than MIN_MATCH: no dictionary lookup


def seqs_of(c, frame=0, block=-1):
    return parsed(c)[frame][block][1]


def by_id(name):
    return next(c for c in CASES if c.id == name)


def test_cases_hit_their_rule():
    """Each crafted case produces the sequence its name promises (so a kernel that breaks the rule cannot match the model)."""
    S = cparse.CM_SEED
    for nb in (2, 3):
        assert seqs_of(by_id(f"seed-{nb}blocks-source-{S}-before-segment=CM_SEED"))[0] == (2000, 24, S + 2000)
        assert seqs_of(by_id(f"seed-{nb}blocks-source-{S + 1}-before-segment=CM_SEED+1"))[0] == (2001, 23, S + 2001)
    assert seqs_of(by_id("choice-t1-longer"))[1] == (991, 12, 8000)
    assert seqs_of(by_id("choice-tp-longer"))[1] == (991, 12, 1000)
    assert seqs_of(by_id("choice-equal-smaller-offset"))[1] == (989, 11, 1000)
    s1 = cparse.seg_bounds(20000, 1)[0]
    assert seqs_of(by_id("round-match-at-lane0"))[0][0] == s1 + 320
    assert seqs_of(by_id("round-match-at-lane31"))[0][0] == s1 + 320 + 31
    assert seqs_of(by_id("round-two-matches-one-round")) == [(s1 + 323, 8, s1 + 323 - 400), (9, 10, s1 + 340 - 900)]
    seglen = cparse.BLOCK // cparse.CM_WARPS
    assert seqs_of(by_id("cap-extension-to-e")) == [(seglen - 40, 40, 260)] * cparse.CM_WARPS     # each ends exactly at e
    assert seqs_of(by_id("cap-e-q=CM_CAP")) == [(seglen - 16, 16, 284)] + [(0, 24, 284), (seglen - 40, 16, 284)] * 7
    for n in (5, 15, 16, 17, 47, 48, 49):
        c = next(c for c in CASES if c.id.startswith(f"cap-ml{n}"))
        assert seqs_of(c)[0] == (7000, n, 7000 - 1234)
    assert len(seqs_of(by_id("dense-5-byte-chunks-CSEG_SEQS=3277"))) > 0.9 * cparse.CM_WARPS * (cparse.BLOCK // 8 // 5)
    assert all(b == (b"", []) for b in parsed(by_id("rle-empty-frame"))[0])
    assert [b[0] for b in parsed(by_id("rle-rle-block-between-two"))[0]][1] == "rle"
    assert all(not b[1] for f in parsed(by_id("isolation-second-frame-starts-with-first-tail")) for b in f)
    # dictionary rules
    assert seqs_of(by_id("dict-len5=MIN_MATCH"))[0] == (0, 5, 5) and seqs_of(by_id("dict-len4=MIN_MATCH-1")) == []
    assert [s[2] for s in seqs_of(by_id("dict-longer-than-WINDOW-head-and-tail"))] == [9000 + 5000]   # not the head's
    assert [s[2] for s in seqs_of(by_id("dict-offset=WINDOW-and-WINDOW+1"))] == [cparse.WINDOW]
    assert [ml for _, ml, _ in seqs_of(by_id("dict-ends-at-dict-end-16-17-40"))[::2]] == [16, 17, 40]
    assert seqs_of(by_id("dict-in-frame-as-long-as-dict"))[1][2] == 19900
    assert seqs_of(by_id("dict-twice-in-dict-later-wins")) == [(700, 24, 700 + 3000 - 2500)]
    assert seqs_of(by_id("dict-no-lookup-in-second-block")) == []
    c5 = by_id("data-c5-200-pieces-raw-content")
    assert sum(1 for f, d in zip(parsed(c5), c5.frames) for b in f for s in b[1] if s[2] > 0) > 200


def test_counts_leave_out_rle_and_cut_long_samples():
    rng = random.Random(5)
    content = bytes(rng.getrandbits(8) for _ in range(3000))
    long = bytes(rng.getrandbits(8) for _ in range(cparse.BLOCK + 500))
    a = cparse.counts([long], content)
    assert (a == cparse.counts([long[:cparse.BLOCK]], content)).all()
    assert int(a[:256].sum()) == cparse.BLOCK
    assert (cparse.counts([b"", b"q" * 5000], content) == 0).all()
    sample = b"x" + content[-40:] + b"y"
    c = cparse.counts([sample], content)
    nseq = len(cparse.parse([sample], content)[0][0][1])       # the 40-byte match, cut at the 6-byte segments' ends
    assert int(c[:256].sum()) == 2 and nseq > 1
    assert int(c[cparse.DS_LL:cparse.DS_ML].sum()) == int(c[cparse.DS_ML:cparse.DS_OF].sum()) == int(c[cparse.DS_OF:].sum()) == nseq


def test_xxh64(oracle):
    assert cparse.xxh64(b"") == 0xEF46DB3751D8E999
    assert cparse.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert cparse.xxh64(b"abc") == 0x44BC2CF5AD770999
    assert cparse.xxh64(b"Nobody inspects the spammish repetition") == 0xFBCEA83C8A378BF1
    rng = random.Random(7)
    for n in list(range(0, 70)) + [255, 256, 1023, 1024, 1025, 32 * 1025 + 31]:
        d = bytes(rng.getrandbits(8) for _ in range(n))
        assert cparse.xxh64(d) == oracle.xxh64(d), n

