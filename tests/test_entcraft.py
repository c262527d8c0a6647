"""CPU checks of the crafted entropy sections (tests/entcraft.py) the GPU tests decode: every case agrees three ways -- the
requested content, the oracle (whose trace must hold exactly the requested literals and sequences) and libzstd -- and invalid
cases fail in the oracle.  Every table description the cases carry is read back by the plain reader, and the RFC 8878 reference
tables are checked entry by entry against the oracle's table builders."""
import ctypes as C
import os

import pytest

import datagen
import entcraft as E

pytestmark = pytest.mark.skipif(not os.path.exists(E.S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def crafted():
    return {g: E.cases(g) for g in E.GROUPS}


@pytest.mark.parametrize("group", list(E.GROUPS))
def test_three_way_agreement(oracle, crafted, group):
    for c in crafted[group]:
        got, err = E.oracle_decode(oracle, c)
        if c.valid:
            assert err is None and got == c.expected, (c, err)
            if c.libzstd:
                assert datagen.decompress(c.frame, len(c.expected), raw_dict=c.dict_raw) == c.expected, c
        else:
            assert err is not None, (c, "the oracle decoded an invalid case")


def _oracle_fse(oracle, norm, log, max_symbol):
    p = (C.c_int32 * len(norm))(*norm)
    out = (C.c_uint32 * (3 << log))()
    assert oracle.lib().zo_kat_fse_build(p, len(norm), log, max_symbol, out) == 0
    return [(int(out[3 * i + 2]), int(out[3 * i + 1]), int(out[3 * i])) for i in range(1 << log)]


def _oracle_huf(oracle, desc):
    mb, ent = C.c_uint8(), (C.c_uint16 * 2048)()
    used = oracle.lib().zo_kat_huf_build(desc, len(desc), C.byref(mb), ent, 2048)
    assert used == len(desc), used
    return mb.value, [(e & 0xFF, e >> 8) for e in ent[:1 << mb.value]]


@pytest.mark.parametrize("group", [g for g in E.GROUPS if g != "errors"])
def test_descriptions_round_trip_and_match_the_oracle(oracle, crafted, group):
    """The reader parses every written description back to the requested counts / weights, and the reference table of every
    description equals the oracle's, entry by entry."""
    n = 0
    for c in crafted[group]:
        for d in c.descriptions():
            n += 1
            if d[0] == "huf":
                h = d[1]
                desc = h.bytes()
                assert E.read_huf_desc(desc) == (h.weights, len(desc)), c
                assert _oracle_huf(oracle, desc) == h.table, c
            else:
                kind, log, norm = d
                data = E.write_ncount(norm, log)
                assert E.read_ncount(data + b"\0") == (log, norm, len(data)), c   # a reader takes whole fields: room for one
                assert _oracle_fse(oracle, norm, log, E.MAX_SYM[kind]) == E.fse_table(norm, log), c
    assert n > 0


def test_predefined_reference_tables(oracle):
    for kind in E.KINDS:
        log, norm = E.PREDEF[kind]
        assert _oracle_fse(oracle, norm, log, E.MAX_SYM[kind]) == E.fse_table(norm, log)


def test_groups_cover_their_edges(crafted):
    """The cases sit where their ids say."""
    huf = [b.huf for c in crafted["huf-tables"] for b in c.blocks if isinstance(b, E.Blk)]
    assert {h.table[0] for h in huf} >= set(range(1, 12))
    nsym = {len(set(s for s, _ in h.table[1])) for h in huf}
    assert nsym >= {2, 31, 32, 33, 64, 65, 96, 97, 128, 129, 200, 255, 256}
    assert any(sorted(h.lengths) == [0, 255] for h in huf) and any(len(h.weights) == 255 for h in huf)
    direct = {len(h.weights) for h in huf if h.desc[0] == "direct"}
    assert direct >= {1, 2, 15, 16, 127, 128}
    fw = {(h.desc[1], any(p == -1 for p in h.desc[2]), len(h.weights) % 2) for h in huf if h.desc[0] == "fse"}
    assert fw >= {(log, neg, odd) for log in (5, 6) for neg in (False, True) for odd in (0, 1)}
    streams = crafted["huf-streams"]
    regen1 = {len(b.lits) for c in streams for b in c.blocks if isinstance(b, E.Blk) and b.streams == 1}
    assert regen1 >= {1, 2, 1022, 1023}
    regen4 = {len(b.lits) for c in streams for b in c.blocks if isinstance(b, E.Blk) and b.streams == 4}
    assert regen4 >= set(range(1, 17)) | {E.S.BLOCK_MAX}
    assert {((len(b.lits) + 3) // 4) % 16 for c in streams if "residue16" in c.id for b in c.blocks if isinstance(b, E.Blk)} == set(range(16))
    for c in streams:
        if c.id.startswith("huf-streams-stream-bytes"):
            pay = E.lit_payload(c.blocks[0].huf.table, c.blocks[0].lits, 4)
            sizes = list(E.struct.unpack("<3H", pay[:6]))
            assert set(sizes + [len(pay) - 6 - sum(sizes)]) == {int(c.id.rsplit("bytes", 1)[1])}, c
    fse = {}
    for c in crafted["fse-tables"]:
        for kind, log, norm in c.descriptions():
            fse.setdefault(kind, []).append((log, norm))
    for kind in E.KINDS:
        got = fse[kind]
        assert {log for log, _ in got} == set(range(5, E.MAX_LOG[kind] + 1)), kind
        assert any(len(n) == E.MAX_SYM[kind] + 1 for _, n in got), kind
        assert {len(n) for _, n in got} >= ({31, 32, 33} if kind != "of" else {31, 32}), kind
        assert any(-1 not in n for _, n in got) and any(n.count(-1) == 1 for _, n in got), kind
        assert any(n.count(-1) > (1 << log) // 2 for log, n in got), kind
        assert any(max(n) == 1 << log for log, n in got), kind
        assert any(max(n) > 8 and 8 in n and 9 in n for _, n in got), kind
        assert any(max((len(g) for g in E._runs(n)), default=0) >= 25 for _, n in got), kind
        rle = {b.modes[E.KINDS.index(kind)][1] for c in crafted["fse-tables"] for b in c.blocks
               if isinstance(b, E.Blk) and b.seqs and b.modes[E.KINDS.index(kind)][0] == "rle"}
        assert E.MAX_SYM[kind] in rle, kind
    assert sum(not c.valid for g in crafted.values() for c in g) >= 25
    assert all(not c.valid for c in crafted["errors"])
