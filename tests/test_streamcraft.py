"""CPU checks of the stream decoder's case set (tests/streamcraft.py): the new cases agree three ways (the model's bytes, the oracle
and, where the format decides, libzstd) and the error cases fail in the oracle where they are meant to; the library's cutter
equals the cut model on every stream at every chunk size; every block boundary is a cut at one chunk size and not at another;
and each stream-edge family hits, at a cut, every residue, stripe remainder, tail size and table kind it is named after.
The crafted cases left out are exactly those the two documented deviations of tier 1d select.  No GPU needed."""
import collections
import os

import pytest

import datagen
import entcraft as E
import seqcraft as S
import streamcraft as SC
import streamcut

pytestmark = pytest.mark.skipif(not os.path.exists(S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def cases():
    crafted = SC.crafted()
    return crafted, SC.new_cases(crafted)


@pytest.fixture(scope="module")
def streams(cases):
    """The valid cases that tier 1d must decode as decode_all_batch does, one stream per group and dictionary set."""
    out = collections.OrderedDict()
    for c in cases[0] + cases[1]:
        if c.valid and not SC.deviation(c):
            out.setdefault((c.group, c.dicts, c.forced.name if c.forced else None), []).append(c)
    return out


def _decoder(oracle, c):
    import dictcraft as D
    d = D.oracle_decoder(oracle) if c.dicts == "dictcraft" else oracle.FrameDecoder()
    if c.dict_raw is not None:
        d.add_dict(c.dict_raw)
    return d


def _oracle(oracle, c):
    """(content or None, (error leaf, stage) or None, blocks decoded before the error)."""
    d = _decoder(oracle, c)
    r = d.reset(c.frame)
    try:
        while not d.is_finished():
            d.decode_blocks(r, oracle.UPTO_BLOCKS, 1)
        return d.collect(), None, d.blocks_decoded()
    except oracle.OracleError as e:
        return None, (oracle.error_names()[e.code].replace("ZO_", ""), e.stage), d.blocks_decoded()


def test_new_cases_three_way(oracle, cases):
    crafted, new = cases
    for c in new:
        if c.kind == "spliced":
            continue
        if c.kind == "ent":
            got, err = E.oracle_decode(oracle, c.src)
        else:
            got, err = S.oracle_decode(oracle, c.frame, c.src.blocks if c.kind == "seq" else c.blocks, c.kind == "seqframe" or c.src.ov)
        if c.valid:
            assert err is None and got == c.expected, (c, err)
            assert len(got) == sum(c.sizes), c
            if c.libzstd:
                assert datagen.decompress(c.frame, len(c.expected), raw_dict=c.dict_raw) == c.expected, c
        else:
            assert err is not None, (c, "the oracle decoded an invalid case")
    for lead, plain in [(c.lead, c.lead_plain) for c in new if c.lead] + [(SC.lead_frame(SC.PHASE_PLAIN), SC.PHASE_PLAIN)]:
        assert oracle.decode_frame(lead)[0] == plain and lead[-4:] == (oracle.xxh64(plain) & 0xFFFFFFFF).to_bytes(4, "little")
    after = [c for c in new if c.group == "errors-after-cut"]
    assert len(after) >= 15
    for c in after:
        # the same error leaf and stage as the crafted case it extends, in the same block, with a block after it
        _, err, nb = _oracle(oracle, c)
        _, err0, nb0 = _oracle(oracle, c.origin)
        assert err == err0 and nb == nb0 == c.fail_block and c.fail_block + 1 < len(c.blocks), (c, err, err0, nb, nb0)


def test_exclusions_are_the_two_deviations(oracle, cases):
    """A crafted case is left out iff one of its sequences reaches past the window or one of its Compressed blocks decodes to
    more than min(128 KiB, window) -- checked for the valid cases against the oracle's trace (actual offsets, block sizes)."""
    crafted, _ = cases
    excluded = [c for c in crafted if SC.deviation(c)]
    for c in crafted:
        if not c.valid:
            continue
        d = _decoder(oracle, c)
        d.trace_enable()
        r = d.reset(c.frame)
        if c.forced is not None:
            d.force_dict(c.forced.id)
        d.decode_blocks(r, oracle.ALL)
        blocks, _, seqs = d.trace()
        assert d.window_size() == c.window, c
        past = any(int(s[3]) > c.window for s in seqs)
        big = any(b["block_type"] == 2 and b["out_size"] > min(SC.BLOCK_MAX, c.window) for b in blocks)
        assert bool(SC.deviation(c)) == (past or big), (c, past, big)
        assert [int(s[3]) for s in seqs] == SC.offsets(c.blocks, c.reps), c
    why = collections.Counter(SC.deviation(c) for c in excluded)
    print(f"{len(excluded)} of {len(crafted)} crafted cases left out: {dict(why)}")
    assert len(excluded) < len(crafted) // 4


@pytest.mark.parametrize("chunk", SC.CHUNKS)
def test_cuts_equal_the_model(pkg, streams, chunk):
    for key, cs in streams.items():
        data = SC.stream(cs, chunk, for_cut=True)[0]
        want, wend = streamcut.cut(data, chunk)
        got, end = pkg.binding.stream_cut(data, chunk)
        got = [tuple(int(r[k]) for k in ("start", "end", "in_bytes", "out_bound", "nblocks", "nseq", "nframes", "flags")) for r in got]
        assert got == want, (key, chunk)
        assert end["status"] == 0 and wend["status"] is None and end["error_offset"] == len(data), (key, chunk, end)
        if chunk == SC.DEFAULT:
            assert len(want) == 1, key


def _all_spans(streams):
    """{case id: {chunk: [(submission flags, [block indices])]}}, {(case id, chunk): [Carry]}."""
    spans, carries = collections.defaultdict(dict), {}
    for key, cs in streams.items():
        for chunk in SC.CHUNKS:
            subs = streamcut.cut(SC.stream(cs, chunk, for_cut=True)[0], chunk)[0]
            car, sp = SC.carries(cs, chunk, subs)
            for cid, lst in sp.items():
                spans[cid][chunk] = [(subs[s][7], ks) for s, ks in lst]
            for cid, lst in car.items():
                carries[(cid, chunk)] = lst
    return spans, carries


@pytest.fixture(scope="module")
def plan(streams):
    return _all_spans(streams)


def test_every_boundary_cut_somewhere_and_inside_somewhere(streams, plan):
    """Every block boundary of every case is a cut at one chunk size and lies inside a submission at another, and a case of three
    or more blocks has a submission that resumes and continues it.  A submission that does so with two or more of the case's
    blocks needs four blocks or more (a frame of three has only its middle block between its first and its last); the count of
    such cases is printed, and the cta-shape family, built for it, must have one."""
    spans, _ = plan
    short, four = [], 0
    for cs in streams.values():
        for c in cs:
            n = len(c.blocks)
            for k in range(1, n):
                cut_at = {ch for ch, sp in spans[c.id].items() if any(ks[0] == k for _, ks in sp)}
                assert cut_at and cut_at != set(SC.CHUNKS), (c, k, cut_at)
            both = [len(ks) for sp in spans[c.id].values() for fl, ks in sp if fl == 3]
            if n >= 3:
                assert both, c
            if n >= 4:
                four += 1
                if max(both) < 2:
                    short.append(c.id)
    print(f"{four - len(short)} of {four} cases of four or more blocks have a submission that resumes and continues them with two "
          f"or more of their blocks; not: {short}")
    assert not [c for c in short if c.startswith("cta-shape")]


def _family(streams, group):
    return [c for key, cs in streams.items() if key[0] == group for c in cs]


def _carries(plan, c):
    return [(ch, x) for ch in SC.CHUNKS for x in plan[1].get((c.id, ch), [])]


def test_table_kinds_carried(streams, plan):
    """Every table, in every kind the carry can hold it, is read by the block right after a cut."""
    got = set()
    for c in _family(streams, "carry-tables"):
        for _, x in _carries(plan, c):
            got |= {(t,) + k for t, k in x.tables.items()}
    want = {("huf", "slot", "huf"), ("huf", "carry", "huf"), ("huf", "dictionary", "dict")}
    for t in ("ll", "of", "ml"):
        want |= {(t, "slot", "fse"), (t, "slot", "rle"), (t, "predefined", "pre"), (t, "carry", "fse"), (t, "dictionary", "dict")}
    assert want <= got, want - got
    cs = {c.id.split("carry-tables-", 1)[1]: c for c in _family(streams, "carry-tables")}
    for streams_n in (1, 4):
        c = cs[f"treeless-{streams_n}stream"]
        assert any(x.next_block == 1 and x.tables.get("huf") == ("slot", "huf") for _, x in _carries(plan, c)), c
    mix = [x.tables for _, x in _carries(plan, cs["ll-new-of-ml-kept"])]
    assert {"ll": ("slot", "fse"), "of": ("carry", "fse"), "ml": ("carry", "fse")} in mix, mix
    # Treeless and Repeat read from the carry slot at three cuts in a row (the slot feeds itself)
    run = sorted(x.next_block for ch, x in _carries(plan, cs["treeless-repeat-over-4-cuts"])
                 if ch == 4096 and set(x.tables.values()) == {("carry", "huf"), ("carry", "fse")})
    assert len(run) >= 3, run
    dct = [x for _, x in _carries(plan, cs["dictionary-tables-by-repeat"]) if x.next_block == 1]
    assert dct and all(set(x.tables.values()) == {("dictionary", "dict")} and len(x.tables) == 4 for x in dct)


def test_history_carried(streams, plan):
    """The first block after a cut starts with repeat codes (the history came across the cut), and the exact-path block sits
    right after one cut and right before the next."""
    for c in _family(streams, "carry-history"):
        cuts = {x.next_block for ch, x in _carries(plan, c) if ch == 4096}
        exact = [k for k, b in enumerate(c.blocks) if b[0] == "cmp" and any(q[0] >= 32768 and q[1] >= 32771 for q in b[2])]
        if exact:
            assert {exact[0], exact[0] + 1} <= cuts, (c, cuts)
            assert exact[0] + 1 < len(c.blocks) and c.blocks[exact[0] + 1][2][0][2] <= 3, c
        else:
            assert 1 in cuts and c.blocks[1][2][0][2] <= 3, c


def test_tail_reach(streams, plan):
    """Each reach right after a cut, with the frame resumed in the submission before the cut, and following its lead frame in
    it; T is the window (1 KiB) or the produced bytes (128 KiB window)."""
    for c in _family(streams, "tail-reach"):
        at = [x for _, x in _carries(plan, c) if x.next_block == 3]
        assert any(x.resumed for x in at), c
        if c.lead:
            assert any(not x.resumed and x.out_off == len(c.lead_plain) for x in at), c
        assert all(x.T == (x.keep if c.window == 1024 else x.P) for x in at), c


def test_alignment_residues_and_stripes(streams, plan):
    res_resumed, res_after_lead = set(), set()
    for c in _family(streams, "align-residue"):
        for _, x in _carries(plan, c):
            assert x.T == x.keep == 1024
            (res_resumed if x.resumed else res_after_lead if x.out_off else set()).add(x.residue)
    assert res_resumed == set(range(16)) and res_after_lead == set(range(16)), (res_resumed, res_after_lead)
    by_t = collections.defaultdict(set)
    for c in _family(streams, "align-stripe"):
        for _, x in _carries(plan, c):
            by_t["window" if x.T == x.keep else "produced"].add(x.unhashed)
    assert by_t["window"] == set(range(32)) and by_t["produced"] == set(range(32)), by_t
    small = [x for c in _family(streams, "align-small") for _, x in _carries(plan, c) if x.P < 32]
    assert {x.P for x in small} >= {1, 2, 15, 16, 17, 31} and all(x.T == x.P for x in small)
    print(f"residues mod 16 at a cut: resumed {sorted(res_resumed)}, after a lead {sorted(res_after_lead)}; "
          f"unhashed bytes mod 32: {len(by_t['window'])} with T = window, {len(by_t['produced'])} with T = produced")


def test_alignment_windows_and_empty_blocks(streams, plan):
    cs = {c.id.split("align-window-", 1)[1]: c for c in _family(streams, "align-window")}
    for n in (12, 21, 31):
        c = cs[f"single-segment-content{n}"]
        assert c.window == n
        xs = [x for _, x in _carries(plan, c)]
        assert xs and all(x.keep == 32 and x.T == x.P < 32 for x in xs), c
    c = cs["single-segment-window1000"]
    assert c.window == 1000 and any(x.T == x.P and x.P % 16 for _, x in _carries(plan, c))
    c = cs["w1024-T=window-produced6144"]
    assert any(x.T == 1024 and x.P >= 6 * 1024 for _, x in _carries(plan, c))
    for name in ("zero-byte-raw-before-cut", "zero-byte-compressed-before-cut", "zero-byte-blocks-over-3-cuts"):
        c = cs[name]
        assert any(c.sizes[x.next_block - 1] == 0 for ch, x in _carries(plan, c) if ch == 4096), c


def test_cta_shape(streams, plan):
    """A submission holds a resumed frame with two or more blocks and >= 4096 compressed bytes (k_exec_cta's eligibility)."""
    spans, _ = plan
    for c in _family(streams, "cta-shape"):
        csize = [n for _, _, n, _ in SC.frame_blocks(c.frame)]
        assert c.dicts is None
        assert any(fl & 1 and len(ks) >= 2 and sum(csize[k] for k in ks) >= 4096 for sp in spans[c.id].values() for fl, ks in sp), c


def test_errors_after_cut_placement(cases):
    """At 4096 the failing block is alone in its submission, after a cut, and the frame goes on past it."""
    after = [c for c in cases[1] if c.group == "errors-after-cut"]
    for c in after:
        data, _, at = SC.stream([c], 4096, for_cut=True)
        subs, end = streamcut.cut(data, 4096)
        # the cutter does not see table errors; each block of the frame is a submission, and the one after the failing block
        # resumes the frame
        frame_subs = subs[-len(c.blocks):]
        assert all(s[4] == 1 for s in frame_subs), c
        assert frame_subs[c.fail_block][7] == 3 and frame_subs[c.fail_block + 1][7] & 1, c
