"""The decoder's dictionary and window reach on crafted frames (tests/dictcraft.py): matches into a dictionary at its edges, the
total_output_counter rule, a dictionary's repeat offsets, reaches at k_exec's batch boundaries and across k_fse's exact-path
replay, offsets past the window, several dictionaries in one submission and forced dictionaries, and output capacities ending
inside a dictionary copy.  Every case runs with both execution kernels: in one batch, one frame per submission, through
FrameDecoder (with the drain schedules in lockstep with the oracle), StreamingDecoder and decode_all.  The bytes must be the
model's, error cases must fail with the model's error leaf and stage, and no frame may write past its out_cap."""
import random

import numpy as np
import pytest

import dictcraft as D

pytestmark = pytest.mark.gpu
CANARY = 0xAB


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def crafted():
    return D.cases()


@pytest.fixture(scope="module")
def dicts(pkg, ctx):
    return {d.name: (pkg.Dictionary.decode_dict(ctx, d.raw) if d.formatted else pkg.Dictionary.raw_content(ctx, d.id, d.content))
            for d in D.DICTS}


@pytest.fixture
def checksummed(pkg, ctx):
    old = ctx.L.b200z_ctx_flags(ctx.h)
    ctx.set_flags(old | pkg.binding.FLAG_CHECKSUM)
    yield
    ctx.set_flags(old)


def _layout(pkg, cs):
    """One slot per frame, 128-byte aligned, with at least 64 canary bytes after each out_cap."""
    io = np.zeros(len(cs), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, c in enumerate(cs):
        io[i] = (so, len(c.frame), oo, c.cap)
        so += len(c.frame)
        oo = (oo + c.cap + 64 + 127) & ~127
    return io, np.frombuffer(b"".join(c.frame for c in cs), dtype=np.uint8), oo


def _check(pkg, cs, io, res, out):
    names = pkg.error_names()
    for i, c in enumerate(cs):
        r, o, want = res[i], int(io[i]["out_off"]), c.batch
        if want.err is None:
            assert r["status"] == 0, (c, names[int(r["status"])], int(r["stage"]))
            assert r["out_size"] == len(want.out) and r["bytes_read"] == len(c.frame), (c, r)
            assert out[o:o + len(want.out)].tobytes() == bytes(want.out), c
            assert r["has_checksum"] and r["has_calculated_checksum"] and r["calculated_checksum"] == r["checksum_from_data"], c
        else:
            assert (names[int(r["status"])].replace("B200Z_", ""), int(r["stage"])) == want.err, (c, r)
        end = o + int(io[i]["out_cap"])
        nxt = int(io[i + 1]["out_off"]) if i + 1 < len(cs) else len(out)
        assert (out[end:nxt] == CANARY).all(), (c, "written past out_cap")


def _run(pkg, ctx, dicts, cs, forced=None):
    import torch
    io, comp, total = _layout(pkg, cs)
    d_out = torch.full((total,), CANARY, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, comp, io, dicts=list(dicts.values()), forced_dict=dicts[forced.name] if forced else None)
    b.run(d_out)
    res = b.finish()
    _check(pkg, cs, io, res, d_out.cpu().numpy())
    return b


def _by_forced(cs):
    out = {}
    for c in cs:
        out.setdefault(c.forced.name if c.forced else None, []).append(c)
    return out


def test_dictcraft_one_batch(pkg, ctx, dicts, crafted, exec_mode, checksummed):
    """All cases in one submission (the forced ones in one more per forced dictionary).  No dictionary frame goes to
    k_exec_cta, and of the frames it takes only the error cases are handed back, for a failed sequence check."""
    for forced, cs in _by_forced(crafted).items():
        b = _run(pkg, ctx, dicts, cs, D.DICTS[[d.name for d in D.DICTS].index(forced)] if forced else None)
        sched = b.debug_sched()
        plain = [c for c in cs if c.use is None]
        if exec_mode == "cta":
            back = [c for c in plain if c.handback]
            assert sched["cta_frames"] == len(plain), sched
            assert sched["handed_back_frames"] == len(back), sched
            assert sched["reasons"] == (D.WHY_SEQ_CHECK if back else 0), sched
        else:
            assert sched["cta_frames"] == 0
        b.close()


def test_dictcraft_one_frame_per_submission(pkg, ctx, dicts, crafted, exec_mode, checksummed):
    for c in crafted:
        b = _run(pkg, ctx, dicts, [c], c.forced)
        sched = b.debug_sched()
        if exec_mode == "cta" and c.use is None:
            assert sched["cta_frames"] == 1 and sched["handed_back_frames"] == (1 if c.handback else 0), (c, sched)
            if c.handback:
                assert sched["reasons"] & c.handback, (c, sched)
        else:
            assert sched["cta_frames"] == 0, (c, sched)
        b.close()


def _decoder(pkg, ctx):
    dec = pkg.FrameDecoder(ctx)
    for d in D.DICTS:
        if d.formatted:
            dec.add_dict(d.raw)
        else:
            dec.add_raw_content_dict(d.id, d.content)
    return dec


def test_dictcraft_frame_decoder(pkg, ctx, crafted, exec_mode):
    names = pkg.error_names()
    for c in crafted:
        dec = _decoder(pkg, ctx)
        if c.valid:
            r = dec.reset(c.frame)
            if c.forced is not None:
                dec.force_dict(c.forced.id)
            assert dec.decode_blocks(r, pkg.ALL) is True
            assert dec.collect() == c.expected, c
            assert dec.bytes_read_from_source() == len(c.frame) and dec.get_checksum_from_data() == dec.get_calculated_checksum()
        else:
            with pytest.raises(pkg.B200ZError) as e:
                r = dec.reset(c.frame)
                if c.forced is not None:
                    dec.force_dict(c.forced.id)
                dec.decode_blocks(r, pkg.ALL)
            assert (names[e.value.code].replace("B200Z_", ""), e.value.stage) == c.full.err, (c, e.value)


def test_dictcraft_drain_schedules_in_lockstep(pkg, ctx, oracle, crafted, exec_mode):
    """decode_blocks(UptoBlocks, 1) + read per block, on the GPU and on the oracle: the same bytes per read, the same
    can_collect, and an error on the same call."""
    names, onames = pkg.error_names(), oracle.error_names()
    cs = [c for c in crafted if c.drains]
    assert cs
    for c in cs:
        g, o = _decoder(pkg, ctx), D.oracle_decoder(oracle)
        gr, orr = g.reset(c.frame), o.reset(c.frame)
        while not o.is_finished():
            try:
                o.decode_blocks(orr, oracle.UPTO_BLOCKS, 1)
                oerr = None
            except oracle.OracleError as e:
                oerr = (onames[e.code].replace("ZO_", ""), e.stage)
            if oerr is None:
                g.decode_blocks(gr, pkg.UPTO_BLOCKS, 1)
            else:
                with pytest.raises(pkg.B200ZError) as e:
                    g.decode_blocks(gr, pkg.UPTO_BLOCKS, 1)
                assert (names[e.value.code].replace("B200Z_", ""), e.value.stage) == oerr, c
                break
            n = o.can_collect()
            assert g.can_collect() == n, c
            assert g.read(n) == o.read(n), c
        else:
            assert g.is_finished() and g.collect() == o.collect(), c


def test_dictcraft_streaming_decoder(pkg, ctx, oracle, crafted, exec_mode):
    """Seeded random read sizes, read for read against the oracle's StreamingDecoder: the same bytes, or the same error leaf
    and stage.  Reads drain the buffer down to the window, which changes what an offset reaches only in quirk cases; every
    other case must give the model's content."""
    rng = random.Random(0xD1C7)
    names, onames = pkg.error_names(), oracle.error_names()
    for c in crafted:
        if not c.valid or c.forced is not None:
            continue
        dec = _decoder(pkg, ctx)
        gd = pkg.StreamingDecoder(ctx, c.frame, decoder=dec)
        od = oracle.StreamingDecoder(c.frame, decoder=D.oracle_decoder(oracle))
        got, failed = bytearray(), False
        while True:
            n = rng.choice([1, 7, 100, 1000, 5000, 1 << 16])
            try:
                want = od.read(n)
            except oracle.OracleError as e:
                with pytest.raises(pkg.B200ZError) as ge:
                    gd.read(n)
                gerr = (names[ge.value.code].replace("B200Z_", ""), dec.L.b200z_frame_decoder_last_stage(dec.h))
                assert gerr == (onames[e.code].replace("ZO_", ""), e.stage), c
                failed = True
                break
            assert gd.read(n) == want, c
            if not want:
                break
            got += want
        if not c.quirk:
            assert not failed and bytes(got) == c.expected, c


def _concat(cs):
    return b"".join(c.frame for c in cs)


def test_dictcraft_decode_all(pkg, ctx, oracle, dicts, crafted, exec_mode):
    """The valid frames that name their dictionary, concatenated: decode_all from device memory and FrameDecoder.decode_all
    give the model's contents back to back; with one error case in the middle both end as the oracle's decode_all does."""
    import torch
    # (FrameDecoder.decode_all reads a frame out every MiB, which changes what the drained cases' offsets reach)
    good = [c for c in crafted if c.valid and c.forced is None and c.use is not None and c.batch is c.full and not c.drains]
    data = _concat(good)
    want = b"".join(c.expected for c in good)
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_out = torch.empty(len(want) + 64, dtype=torch.uint8, device="cuda")
    summary, res = pkg.decode_all(ctx, d_in, d_out, dicts=list(dicts.values()))
    assert summary["status"] == 0 and summary["frames"] == len(good) and summary["written"] == len(want), summary
    assert d_out[:len(want)].cpu().numpy().tobytes() == want
    assert _decoder(pkg, ctx).decode_all(data, len(want)) == want

    bad = next(c for c in crafted if not c.valid and c.use is not None and c.forced is None)
    k = len(good) // 2
    chain = good[:k] + [bad] + good[k:]
    data = _concat(chain)
    cap = sum(len(c.expected) if c.valid else c.cap for c in chain)
    names, onames = pkg.error_names(), oracle.error_names()
    with pytest.raises(oracle.OracleError) as oe:
        D.oracle_decoder(oracle).decode_all(data, cap)
    oleaf = onames[oe.value.code].replace("ZO_", "")
    d_out = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    summary, res = pkg.decode_all(ctx, torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(), d_out, dicts=list(dicts.values()))
    assert names[summary["status"]].replace("B200Z_", "") == oleaf and summary["error_frame"] == k, summary
    before = b"".join(c.expected for c in good[:k])
    assert summary["written"] >= len(before) and d_out[:len(before)].cpu().numpy().tobytes() == before, summary
    with pytest.raises(pkg.B200ZError) as ge:
        _decoder(pkg, ctx).decode_all(data, cap)
    assert names[ge.value.code].replace("B200Z_", "") == oleaf
