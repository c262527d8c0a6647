"""The decoder's sequence and execution kernels (k_fse, k_exec, k_exec_cta) on crafted sequence sets (tests/seqcraft.py):
sequence counts around the batch constants, overlapping matches at every row residue, dense ownership, sources in earlier
blocks, blocks at the edges of k_exec_cta's record fields, repeat offsets, and k_fse's fast / exact path boundary.  Every case
runs with both execution kernels, all cases in one batch and one frame per submission; the bytes must be the plain LZ77
reference's, error cases must fail with the oracle's error leaf and stage, and no frame may write past its out_cap."""
import numpy as np
import pytest

import seqcraft as S

pytestmark = pytest.mark.gpu
CANARY = 0xAB


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def crafted(oracle):
    cs = S.cases()
    for c in cs:
        c.err = None if c.valid else S.oracle_decode(oracle, c.frame, c.blocks, c.ov)[1]
    return cs


def _layout(pkg, cs):
    """One slot per frame, 128-byte aligned (so that a case's residues are row residues), with at least 64 canary bytes
    after each out_cap."""
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
        r, o = res[i], int(io[i]["out_off"])
        if c.valid:
            assert r["status"] == 0, (c, names[int(r["status"])], int(r["stage"]))
            assert r["out_size"] == len(c.expected) and r["bytes_read"] == len(c.frame), (c, r)
            assert out[o:o + len(c.expected)].tobytes() == c.expected, c
        else:
            assert (names[int(r["status"])].replace("B200Z_", ""), int(r["stage"])) == c.err, (c, r)
        end = o + int(io[i]["out_cap"])
        nxt = int(io[i + 1]["out_off"]) if i + 1 < len(cs) else len(out)
        assert (out[end:nxt] == CANARY).all(), (c, "written past out_cap")


def _run(pkg, ctx, cs):
    import torch
    io, comp, total = _layout(pkg, cs)
    d_out = torch.full((total,), CANARY, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, comp, io)
    b.run(d_out)
    res = b.finish()
    _check(pkg, cs, io, res, d_out.cpu().numpy())
    return b


def test_crafted_one_batch(pkg, ctx, crafted, exec_mode):
    b = _run(pkg, ctx, crafted)
    sched = b.debug_sched()
    if exec_mode == "cta":
        back = [c for c in crafted if c.handback is not None]
        assert sched["cta_frames"] == len(crafted)
        assert sched["handed_back_frames"] == len(back), sched
        assert sched["reasons"] == np.bitwise_or.reduce([c.handback for c in back]), sched
    else:
        # k_fse: a sequence with more than FSE_FAST_XBITS extra bits sends its block to the exact path (raw offsets)
        assert sched["cta_frames"] == 0
        first = np.cumsum([0] + [len(c.blocks) for c in crafted])
        seen = set()
        for i, c in enumerate(crafted):
            if c.group == "fse" and c.valid:
                raw = bool(b.debug_block_flags(int(first[i])) & 1)
                assert raw == (c.xbits > S.FSE_FAST_XBITS), (c, raw)
                seen.add(c.xbits)
        assert seen == {32, 33, S.FSE_FAST_XBITS, S.FSE_FAST_XBITS + 1}
    b.close()


def test_crafted_one_frame_per_submission(pkg, ctx, crafted, exec_mode):
    for c in crafted:
        b = _run(pkg, ctx, [c])
        if exec_mode == "cta":
            sched = b.debug_sched()
            if c.handback is None:
                assert sched["handed_back_frames"] == 0, (c, sched)
            else:
                assert sched["handed_back_frames"] == 1 and sched["reasons"] & c.handback, (c, sched)
        b.close()


def test_crafted_frame_decoder(pkg, ctx, crafted, exec_mode):
    """A subset through FrameDecoder.decode_blocks: every error case, the 128 KiB blocks, and every third other case."""
    names = pkg.error_names()
    picked = [c for i, c in enumerate(crafted) if not c.valid or c.group in ("cta-block", "fse") or i % 3 == 0]
    for c in picked:
        dec = pkg.FrameDecoder(ctx)
        if c.valid:
            r = dec.reset(c.frame)
            assert dec.decode_blocks(r, pkg.ALL) is True
            assert dec.collect() == c.expected, c
            assert dec.bytes_read_from_source() == len(c.frame) and dec.get_checksum_from_data() == dec.get_calculated_checksum()
        else:
            with pytest.raises(pkg.B200ZError) as e:
                r = dec.reset(c.frame)
                dec.decode_blocks(r, pkg.ALL)
            assert (names[e.value.code].replace("B200Z_", ""), e.value.stage) == c.err, (c, e.value)
