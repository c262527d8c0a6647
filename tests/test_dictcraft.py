"""CPU checks of the crafted dictionary and window-reach frames (tests/dictcraft.py) the GPU tests decode: the model agrees with the
oracle on every case (bytes, or error leaf and stage) and with libzstd wherever the format itself decides; the drain schedules
agree with the oracle read by read; each case marked `quirk` is one where the reference's rules and the format's differ, and no
other is; every group holds the edges its ids name."""
import ctypes as C
import os
import struct

import pytest

import datagen
import dictcraft as D

pytestmark = pytest.mark.skipif(not os.path.exists(D.S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def crafted():
    return {g: D.cases(g) for g in D.GROUPS}


def test_dictionaries_load_as_built(oracle):
    """Every formatted dictionary decodes in the oracle with the ID, repeat offsets and content it was built with."""
    L = oracle.lib()
    for d in D.DICTS:
        if not d.formatted:
            continue
        i, h, n = C.c_uint32(), (C.c_uint32 * 3)(), C.c_size_t()
        assert L.zo_kat_decode_dict(d.raw, len(d.raw), C.byref(i), h, C.byref(n)) == 0, d
        assert (i.value, tuple(h), n.value) == (d.id, d.reps, len(d.content)), d


@pytest.mark.parametrize("group", list(D.GROUPS))
def test_model_and_oracle_agree(oracle, crafted, group):
    for c in crafted[group]:
        got, err = D.oracle_decode(oracle, c)
        if c.full.err is None:
            assert err is None and got == c.expected, (c, err)
        else:
            assert err == c.full.err, (c, err, c.full.err)
        if c.batch is not c.full:       # an output capacity: decode_all into exactly out_cap bytes
            d = D.oracle_decoder(oracle)
            with pytest.raises(oracle.OracleError) as e:
                d.decode_all(c.frame, c.cap)
            assert oracle.error_names()[e.value.code].replace("ZO_", "") == c.batch.err[0], c


@pytest.mark.parametrize("group", list(D.GROUPS))
def test_libzstd_agrees_where_the_format_decides(crafted, group):
    n = 0
    for c in crafted[group]:
        rfc = c.run(rfc=True)
        if rfc.err is not None or c.quirk or not c.libzstd:
            continue
        dic = (c.use.raw if c.use.formatted else c.use.content) if c.use is not None else None
        assert datagen.decompress(c.frame, len(c.expected), raw_dict=dic) == c.expected, c
        n += 1
    assert n > 0 or group in ("nodict",)


def test_drain_schedules(oracle, crafted):
    """decode_blocks(UptoBlocks, 1) + read per block on the oracle; the model, given the bytes the oracle read, agrees."""
    cs = [c for g in crafted.values() for c in g if c.drains]
    assert len(cs) >= 2
    for c in cs:
        out, err, drains, _ = D.oracle_drained(oracle, c)
        r = c.run(drains=drains)
        assert err == r.err, (c, err, r.err)
        if err is None:
            assert out == bytes(r.out), c
            assert r.outcome != c.expected or not c.valid, (c, "the reads change nothing")
        else:
            assert c.valid, (c, "the schedule must turn a frame the batch tier accepts into an error")


def test_quirk_cases_are_real(crafted):
    for c in (c for g in crafted.values() for c in g):
        ref, rfc = c.full.outcome, c.run(rfc=True).outcome
        assert (ref != rfc) == c.quirk, (c, "quirk" if c.quirk else "not a quirk", ref is D.ERROR, rfc is D.ERROR)


def _by_id(cs):
    return {c.id.split("-", 1)[1]: c for c in cs}


def test_every_named_edge_is_present(crafted):
    reach = _by_id(crafted["reach"])
    dl = len(D.D_MAIN.content)
    r = reach["of=produced+dict_len"].full.reaches
    assert r[0][3] == dl and r[0][4] == "full"
    assert reach["of=produced+dict_len+1"].full.err[0] == D.NOT_IN_DICT and reach["of=produced+dict_len+1"].full.reaches[-1][3] == dl + 1
    for name, kind, delta in (("from_dict=ml-full", "full", 0), ("from_dict=ml-1-straddle-by-one", "straddle", -1), ("from_dict=ml+1-full", "full", 1)):
        (b, si, _, fd, k), = reach[name].full.reaches
        assert k == kind and fd - reach[name].blocks[b][2][si][1] == delta, name
    (b, si, _, fd, k), = reach["straddle-at-frame-start-periodic"].full.reaches
    assert (b, si, k) == (0, 0, "straddle") and reach["straddle-at-frame-start-periodic"].blocks[0][2][0][1] - fd > fd
    assert reach["one-byte-dict-straddle"].full.reaches[0][3:] == (1, "straddle")
    assert reach["one-byte-dict-of=produced+2"].full.err[0] == D.NOT_IN_DICT
    assert len(D.D_LONG.content) > reach["dict-longer-than-window"].window
    assert reach["straddle-after-read-drained"].drains

    for c in crafted["counter"]:
        if "counter=" in c.id:
            W = c.window
            if c.id.endswith("=W"):
                assert c.valid and max(x[2] for x in c.full.reaches) == W, c
            else:
                assert c.full.err[0] == D.TOO_BIG and c.full.fail[2] == W + 1, c
    assert {c.window for c in crafted["counter"] if "counter=" in c.id} == {1024, 1408}
    cnt = _by_id(crafted["counter"])
    for name in ("rle-100KiB-then-reach", "raw-100KiB-then-reach", "full-copies-1500-uncounted"):
        assert cnt[name].valid and any(k for *_, k in cnt[name].full.reaches), name
    full = [x for x in cnt["full-copies-1500-uncounted"].full.reaches if x[4] == "full"]
    assert sum(cnt["full-copies-1500-uncounted"].blocks[0][2][x[1]][1] for x in full[:-1]) > cnt["full-copies-1500-uncounted"].window
    assert sum(c.single_segment for c in crafted["counter"]) == 2

    reps = _by_id(crafted["reps"])
    for ov in (1, 2, 3):
        for ll in (0, 5):
            c = reps[f"ov{ov}-ll{ll}-into-content"]
            assert c.valid and c.full.reaches[0][:2] == (0, 0), c
    assert reps["rep0=1-ov3-ll0-offset0"].full.err[0] == "ERR_EXEC_ZERO_OFFSET"
    for name in D.REP_VALUES:
        for slot in range(3):
            for sep in ("first", "after-raw", "after-rle", "after-cmp0seq"):
                c = reps[f"rep{slot}={name}-ll4-{sep}"]
                b = len(c.blocks) - 1
                assert c.full.fail is None or c.full.fail[:2] == (b, 0), c      # it fails, if at all, on the value itself
        assert f"rep0={name}-unused" in reps

    bt = _by_id(crafted["batch"])
    for idx in (0, 63, 64, 65, 127, 128):
        c = bt[f"reach-at-seq{idx}"]
        assert [x[1] for x in c.full.reaches] == [idx] and c.valid, c
    assert {c.xbits for c in crafted["batch"] if hasattr(c, "xbits")} == {D.FSE_FAST_XBITS, D.FSE_FAST_XBITS + 1}
    for c in crafted["batch"]:
        if hasattr(c, "xbits"):
            assert c.valid and {x[4] for x in c.full.reaches} == {"full", "straddle"}, c

    nd = crafted["nodict"]
    flips = {c.id: c.full for c in nd if "counter=" in c.id}
    assert len(flips) == 4
    for cid, r in flips.items():
        assert r.err[0] == (D.NOT_IN_DICT if cid.endswith("=W") else D.TOO_BIG) and r.fail[2] == 1024 + (0 if cid.endswith("=W") else 1), cid
    past = _by_id(nd)["of-past-window-inside-produced"]
    assert past.valid and past.window < 2000 and not past.full.reaches

    m = crafted["multi"]
    assert {(c.use.name, c.id_bytes) for c in m if c.forced is None} == {(d.name, b) for d in (D.D_A, D.D_R) for b in (1, 2, 4)} | {(D.D_B.name, 2), (D.D_B.name, 4)}
    assert any(c.forced is not None and c.dict is not None and c.forced is not c.dict for c in m)
    for c in crafted["cap"]:
        (b, si, _, fd, k), = c.full.reaches
        ml = c.blocks[b][2][si][1]
        assert c.batch.err == ("ERR_TARGET_TOO_SMALL", D.STAGE_DRAIN) and c.valid
        at = c.cap - len(c.batch.out)       # bytes of the copy that fit
        assert 0 < at < ml and ((k == "full") or at > fd), c


def _window_buffer_moves(blocks, drains):
    """The window buffer of a decoder that submits one block at a time and keeps the frame from `base` on, in a buffer that grows
    to max(live + block + 64, 1.5 x its size, 1 MiB) and drops the drained bytes (base = drained) when a block does not fit.
    Returns the indices of the blocks that moved it, and per block the (base, drained) it executes with."""
    cap = base = produced = drained = 0
    moves, at = [], []
    for i, b in enumerate(blocks):
        extra = D.S.nominal_size([b])
        if produced - base + extra + 64 > cap:
            cap = max(produced - drained + extra + 64, cap + cap // 2, 1 << 20)
            base = drained
            moves.append(i)
        at.append((base, drained))
        produced += extra
        drained += drains[i]
    return moves, at


def test_straddles_follow_window_buffer_moves(oracle, crafted):
    """The multi-MiB drained case: read block by block, the window buffer moves at least three times, and after every move but
    the first (which starts from nothing drained) a straddle executes with bytes drained past the buffer's new start, so its
    second part is read at an offset inside the moved buffer."""
    c = _by_id(crafted["reach"])["straddle-after-read-window-buffer-growth-drained"]
    _, err, drains, _ = D.oracle_drained(oracle, c)
    assert err is None
    r = c.run(drains=drains)
    straddles = {b for b, _, _, _, k in r.reaches if k == "straddle"}
    assert len(straddles) == sum(b[0] == "cmp" for b in c.blocks)
    moves, at = _window_buffer_moves(c.blocks, drains)
    assert len(moves) >= 3, moves
    for m, nxt in zip(moves[1:], moves[2:] + [len(c.blocks)]):
        assert any(m < b < nxt and at[b][1] > at[b][0] for b in straddles), (m, nxt)
