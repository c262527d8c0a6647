"""The plain model of the OPT level (tests/copt.py) checked against the format, without the GPU: every case's parse replays to its
input within the window, the frame and the segment; the frames reference_frame assembles decode with the oracle and libzstd; the
finder's chain is the brute-force nearest earlier position with the same hash; without repeat candidates the DP's cost on small
segments is an exhaustive search's minimum under the same prices; each crafted case hits the rule it is named after; and on 64
frames of 128 KiB of C2b-shaped text the model's ratio is at least libzstd level 3's and above LAZY's."""
import itertools
import os
import random

import pytest

import clazy
import copt
import cparse
import datagen
import seqcraft

pytestmark = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")
CASES = copt.cases()
_parsed = {}


def parsed(c):
    if c.id not in _parsed:
        _parsed[c.id] = cparse.parse(c.frames, c.content, copt.OPT)
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
        for k, b in enumerate(blocks):
            if b[0] == "rle":
                continue
            n = min(cparse.BLOCK, len(data) - k * cparse.BLOCK)
            seglen = -(-n // cparse.CM_WARPS)
            for pos, ml, of in positions(b[1]):
                fpos = k * cparse.BLOCK + pos
                assert ml >= copt.MIN_MATCH and 1 <= of <= copt.WINDOW
                assert pos // seglen == (pos + ml - 1) // seglen, "a match crosses its segment's end"
                if of > fpos:
                    assert k == 0 and of - fpos <= tail and ml <= of - fpos, "a dictionary source past the dictionary's end"


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_reference_frame_decodes(oracle, c):
    for data, blocks in zip(c.frames, parsed(c)):
        f = cparse.reference_frame(data, blocks, level=copt.OPT)
        assert datagen.decompress(f, len(data), raw_dict=c.content) == data
        assert oracle.decode_frame(f, raw_dict=c.content)[0] == data


def brute_prev(H):
    last, out = {}, []
    for q, h in enumerate(H):
        out.append(last.get(h, -1))
        last[h] = q
    return out


def test_chain_is_the_nearest_same_hash_position():
    """Frames of random bytes over small alphabets (many equal hashes), a frame of 3 blocks with repeats at offsets 131072 and
    131073 and from the previous block, and one whose first bytes repeat: prev is the brute-force rule, and the finder never
    walks past offset 131072."""
    rng = random.Random(5)
    frames = [bytes(rng.choice(b"ab") for _ in range(3000)), bytes(rng.choice(b"abcd") for _ in range(5000))]
    big = cparse.rand(rng, 3 * cparse.BLOCK)
    cparse.plant(big, cparse.BLOCK + 100, 100, 40)
    cparse.plant(big, 2 * cparse.BLOCK + 100, cparse.BLOCK + 99, 40)
    cparse.plant(big, 2 * cparse.BLOCK + 9000, 2 * cparse.BLOCK - 3000, 40)
    frames += [bytes(big), b"abcde" * 20]
    for f in frames:
        H = cparse.hashes(f, copt.OPT_HASH_LOG)
        assert copt.chain(H) == brute_prev(H)
    F = bytes(big)
    prev = copt.chain(cparse.hashes(F, copt.OPT_HASH_LOG))
    base = 2 * cparse.BLOCK
    for q in (100, 9000):
        offs = [o for _, o, _ in copt.candidates(F, base, cparse.BLOCK, q, cparse.BLOCK, prev, None, None)]
        assert all(o <= copt.WINDOW for o in offs)
    assert cparse.BLOCK + 1 not in [c[1] for c in copt.candidates(F, base, cparse.BLOCK, 100, cparse.BLOCK, prev, None, None)]
    assert (copt.OPT_CAP, 3000 + 9000) in [c[:2] for c in copt.candidates(F, base, cparse.BLOCK, 9000, cparse.BLOCK, prev, None, None)]


def exhaustive(F, i, stop, cands, lit):
    """The cheapest parse of [i, stop) by enumerating every parse (no memo): literals and matches of the finder's lists."""
    if i == stop:
        return 0
    best = lit[F[i]] + exhaustive(F, i + 1, stop, cands, lit)
    prev_len = copt.MIN_MATCH - 1
    for ln, o, _ in cands(i) if i + copt.MIN_MATCH <= stop else ():
        for l in range(prev_len + 1, ln + 1):
            best = min(best, copt.MATCH_W + copt.of_price(o) + exhaustive(F, i + l, stop, cands, lit))
        prev_len = ln
    return best


@pytest.mark.parametrize("seed", range(6))
def test_dp_cost_is_the_exhaustive_minimum_without_repeats(seed):
    rng = random.Random(seed)
    words = [bytes(rng.getrandbits(8) for _ in range(rng.randint(5, 9))) for _ in range(3)]
    F = bytearray(cparse.rand(rng, 60))
    while len(F) < 60 + 22:
        F += rng.choice(words) if rng.random() < 0.7 else bytes([rng.getrandbits(8)])
    F = bytes(F[:82])
    a, stop = 60, 82
    prev = copt.chain(cparse.hashes(F, copt.OPT_HASH_LOG))
    lit = copt.lit_prices(F)

    def cands(i):
        return copt.candidates(F, 0, 0, i, stop, prev, None, None)
    assert any(cands(i) for i in range(a, stop))
    end, path, _, taken, cost = copt.dp(F, 0, 0, a, stop, (), cands, lit, use_reps=False)
    assert end == stop and taken is None
    assert cost == exhaustive(F, a, stop, cands, lit)
    paid = 0                                                        # the path's matches and literals add up to its cost
    p = a
    for q, ml, o in path:
        paid += sum(lit[F[j]] for j in range(p, q)) + copt.MATCH_W + copt.of_price(o)
        p = q + ml
    assert paid + sum(lit[F[j]] for j in range(p, stop)) == cost


def seqs_at(c, block=-1):
    return positions(parsed(c)[0][block][1])


def test_cases_hit_their_rule():
    s = cparse.seg_bounds(40000, 1)[0]
    assert seqs_at(by_id("suff-ml31=SUFF-1")) == [(s + 700, 31, 3000)]
    assert seqs_at(by_id("suff-ml32=SUFF")) == [(s + 700, 32, 3000)]                                  # taken at once
    assert seqs_at(by_id("suff-ml60=SUFF-extended-to-60")) == [(s + 700, 60, 3000)]                   # and extended
    c = by_id("rep-repeat-along-one-path")
    assert seqs_at(c) == [(9000, 9, 777), (9021, 9, 777)] and clazy.reps(parsed(c)[0][0][1])[1][2] == 1
    assert seqs_at(by_id("rep-cost-tie-smaller-offset")) == [(8000, 12, 12), (9000, 12, 1000)]   # not 1012
    assert seqs_at(by_id(f"chain-offset-{copt.WINDOW}=WINDOW")) == [(5000, 24, copt.WINDOW)]
    assert seqs_at(by_id(f"chain-offset-{copt.WINDOW + 1}=WINDOW+1")) == []
    assert seqs_at(by_id("chain-source-at-frame-start")) == [(2000, 30, 2000)]
    w = seqs_at(by_id(f"wincap-matches-across-W={copt.OPT_WIN}"))
    assert len(w) > 80 and w[0][0] == 6000
    assert parsed(by_id("wincap-literals-only-W"))[0][0][1] == []


def test_dp_closes_at_the_window_cap():
    """Over more than W positions the parse is the DP from each cap onwards: the first DP ends at node a + W exactly."""
    c = by_id(f"wincap-matches-across-W={copt.OPT_WIN}")
    F = c.frames[0]
    n = len(F)
    seglen = -(-n // cparse.CM_WARPS)
    w = 6000 // seglen
    s, e = cparse.seg_bounds(n, w)
    prev = copt.chain(cparse.hashes(F, copt.OPT_HASH_LOG))
    lit = copt.lit_prices(F)

    def cands(i):
        return copt.candidates(F, 0, 0, i, e, prev, None, None)
    end, path, _, taken, _ = copt.dp(F, 0, 0, s, e, (), cands, lit)
    assert taken is None and end == s + copt.OPT_WIN
    assert all(q + ml <= end for q, ml, _ in path)
    assert positions(parsed(c)[0][0][1])[:len(path)] == path


def test_forced_pieces_end_the_dp():
    """A forced piece (tests/cldm.py's kept matches) is one sequence and a repeat; the DPs run up to its start and from its end."""
    rng = random.Random(9)
    buf = cparse.rand(rng, 40000)
    cparse.plant(buf, 20000, 12000, 300)
    cparse.plant(buf, 20400, 20400 - 8000, 12)                      # after the piece, its offset again: a repeat
    F = bytes(buf)
    blocks = cparse.parse_frame(F, copt.OPT, kept=[[(20000, 300, 8000)]])
    seqs = positions(blocks[0][1])
    s1 = cparse.seg_bounds(40000, 4)[0]                             # 20000: segment 4 starts there
    assert s1 == 20000 and (20000, 300, 8000) in seqs and (20400, 12, 8000) in seqs
    recs = clazy.reps(blocks[0][1])
    assert recs[[p for p, _, _ in seqs].index(20400)][2] == 1


def test_ratio_at_least_libzstd_level3():
    """64 frames of 128 KiB of C2b-shaped text: the model's frames against libzstd 1.5.5 level 3 with a 128 KiB window, and LAZY."""
    from concurrent.futures import ProcessPoolExecutor
    plain = datagen.c2_text_plain(64 * 131072).tobytes()
    datas = [plain[i:i + 131072] for i in range(0, len(plain), 131072)]
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:   # parse in parallel, encode here
        blocks = list(ex.map(cparse.parse_frame, datas, itertools.repeat(copt.OPT, len(datas))))
    ratio = len(plain) / sum(len(cparse.reference_frame(d, b, level=copt.OPT)) for d, b in zip(datas, blocks))
    zstd3 = len(plain) / sum(len(datagen.compress(d, level=3, window_log=17)) for d in datas)
    print(f"OPT model ratio {ratio:.3f}, libzstd level 3 {zstd3:.3f}")
    assert ratio >= zstd3 and ratio > 2.698                         # LAZY's on these frames
