"""CPU checks of the crafted invalid frames (tests/errcraft.py) the GPU tests decode, and of the census of the decoder's error leaves:
every case fails in the oracle with the leaf, stage and failing block it names; libzstd rejects it too; the census classifies every
decoding leaf of include/b200zstd.h and every REFERENCE_WOULD_PANIC site of the oracle, so a new leaf or site fails here until someone
classifies it."""
import os
import re

import pytest

import datagen
import errcraft as X

pytestmark = pytest.mark.skipif(not os.path.exists(X.E.S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def crafted():
    return X.cases()


def _oracle_error(oracle, fn):
    try:
        fn()
    except oracle.OracleError as e:
        return oracle.error_names()[e.code].replace("ZO_ERR_", ""), e.stage
    return None


def test_cases_fail_in_the_oracle_with_their_leaf(oracle, crafted):
    for c in crafted:
        d = oracle.FrameDecoder()

        def run():
            r = d.reset(c.frame)
            d.decode_blocks(r, oracle.ALL)
        assert _oracle_error(oracle, run) == (c.leaf, c.stage), c
        if c.stage > X.FRAME_HEADER:
            assert d.blocks_decoded() == c.error_block, c
        # a fault that is not the input ending fails the same way with more bytes after the frame
        if not c.at_end:
            d = oracle.FrameDecoder()
            assert _oracle_error(oracle, lambda: d.decode_blocks(d.reset(c.frame + bytes(64)), oracle.ALL)) == (c.leaf, c.stage), c


def test_libzstd_rejects_every_case(crafted):
    for c in crafted:
        if c.libzstd:
            with pytest.raises(RuntimeError):
                datagen.decompress(c.frame, c.cap)


def test_dictionaries_fail_in_the_oracle(oracle):
    dicts, good = X.dictionaries()
    oracle.FrameDecoder().add_dict(good)
    for name, raw, leaf in dicts:
        assert _oracle_error(oracle, lambda: oracle.FrameDecoder().add_dict(raw)) == (leaf, X.DICTIONARY), name


def test_good_frames_decode(oracle):
    for data, plain in X.good_frames():
        assert oracle.decode_frame(data)[0] == plain


def test_cases_cover_their_variants(crafted):
    ids = {c.id for c in crafted}
    for c in crafted:
        if c.id.endswith("-first"):
            assert c.id[:-len("first")] + "later" in ids, c
    for leaf in ("HUF_SOURCE_IS_EMPTY", "HUF_NOT_ENOUGH_BYTES_IN_SOURCE", "HUF_MISSING_WEIGHTS", "HUF_TOO_MANY_WEIGHTS", "HUF_EXTRA_PADDING"):
        got = {c.id for c in crafted if c.leaf == leaf}
        assert any("1stream" in i for i in got) and any("4stream" in i for i in got), leaf
    assert {"direct", "fse"} <= {w for c in crafted if c.leaf == "HUF_MISSING_WEIGHTS" for w in ("direct", "fse") if w in c.id}
    lit = {c.id for c in crafted if c.leaf == "LIT_BITSTREAM_READ_MISMATCH"}
    assert all(any(f"{w}-weights" in i for i in lit) for w in ("direct", "fse")) and any("treeless" in i for i in lit)
    for kind in ("LL", "OF", "ML"):
        assert any(c.leaf == f"SEQ_MISSING_BYTE_FOR_RLE_{kind}_TABLE" for c in crafted), kind


def test_overshooting_streams_are_what_they_say(crafted):
    """The literal-stream model behind overshooting_stream agrees with the writer on valid streams."""
    h = X.E.Huf(X.E.lengths_for(X.random.Random(5), range(20), 6))
    lits = X.E.literals(X.random.Random(6), h.lengths, 300)
    assert X.huf_decode_stream(h.table, X.E.huf_stream(h.table, lits)) == (list(lits), True)
    bad = X.overshooting_stream(h.table, lits[:40])
    assert not X.huf_decode_stream(h.table, bad)[1]


def test_census_classifies_every_leaf():
    leaves = X.decoding_leaves()
    assert len(leaves) > 60 and leaves["DICT_BAD_MAGIC_NUM"] == 121 and leaves["REFERENCE_WOULD_PANIC"] == 200
    census = X.census()
    missing = sorted(set(leaves) - set(census))
    assert not missing, f"unclassified error leaves: {missing}"
    reached = {leaf for leaf, (how, _) in census.items() if how == "case"}
    # one class per leaf
    for table in (X.COVERED_ELSEWHERE, X.UNREACHABLE, X.NOT_TESTED):
        assert not reached & set(table), reached & set(table)
        assert set(table) <= set(leaves), set(table) - set(leaves)
    assert not set(X.COVERED_ELSEWHERE) & set(X.UNREACHABLE) and not set(X.UNREACHABLE) & set(X.NOT_TESTED)
    # an unreachable leaf shows the oracle's line and the reference's
    for leaf, why in X.UNREACHABLE.items():
        assert re.search(r"ruzstd_oracle\.c:\d+", why) and re.search(r"\w+\.rs:\d+", why), leaf


def test_census_names_existing_tests():
    for leaf, test in X.COVERED_ELSEWHERE.items():
        path, name = test.split("::")
        assert re.search(rf"^def {name}\(", open(os.path.join(X.ROOT, path)).read(), re.M), (leaf, test)


def test_census_classifies_every_reference_panic_site():
    assert X.panic_lines() == sorted(X.PANIC_SITES), "a REFERENCE_WOULD_PANIC site of oracle/ruzstd_oracle.c is not classified"


def test_oracle_and_library_number_the_leaves_alike(oracle):
    zo = {v.replace("ZO_ERR_", ""): k for k, v in oracle.error_names().items() if v.startswith("ZO_ERR_")}
    for leaf, code in X.decoding_leaves().items():
        assert zo.get(leaf) == code, leaf


def test_reentry_cases_reach_their_panic_sites(oracle):
    """Called again after the first error, the oracle's decode_blocks reads the next block and reaches the panic site the census
    credits to the case."""
    sites = {r.site for r in X.reentries()}
    assert sites == {line for line, why in X.PANIC_SITES.items() if why.startswith("REACHED")}
    for r in X.reentries():
        d = oracle.FrameDecoder()
        src = d.reset(r.frame)
        assert _oracle_error(oracle, lambda: d.decode_blocks(src, oracle.ALL)) == r.first, r
        assert _oracle_error(oracle, lambda: d.decode_blocks(src, oracle.ALL)) == r.second, r
        assert "return ZO_ERR_REFERENCE_WOULD_PANIC" in open(X.ORACLE_C).read().splitlines()[r.site - 1], r
