"""The decoder's entropy stage (k_setup's table builders, k_huf's literal streams) on crafted entropy sections
(tests/entcraft.py): Huffman tables of every max_bits and of symbol counts across every 32-lane chunk, direct and FSE-compressed
weight descriptions, 1 and 4 streams at the fast path's edges, Treeless literals, FSE tables at every accuracy log and at the
edges of the description format, Repeat modes, a formatted dictionary, and table / stream errors.

Every case runs with both execution kernels, all cases in one batch and one frame per submission.  For every Compressed block
of a valid case the tables it decoded with are read back and must equal the RFC 8878 reference table of the description that
defined them, entry by entry; its literals and sequences must be the requested ones; the bytes, out_size, bytes_read and the
checksum must be right and nothing may be written past out_cap.  Invalid cases must fail with the oracle's error leaf and stage.
The Treeless, Repeat and dictionary cases also go block by block through FrameDecoder, so that their tables cross submissions."""
import numpy as np
import pytest

import entcraft as E

pytestmark = pytest.mark.gpu
CANARY = 0xAB


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


@pytest.fixture(scope="module")
def crafted(oracle):
    cs = E.cases()
    for c in cs:
        c.err = None if c.valid else E.oracle_decode(oracle, c)[1]
    return cs


@pytest.fixture
def checksummed(pkg, ctx):
    old = ctx.L.b200z_ctx_flags(ctx.h)
    ctx.set_flags(old | pkg.binding.FLAG_CHECKSUM)
    yield
    ctx.set_flags(old)


def _layout(pkg, cs):
    """Frames 16-byte aligned in the input (a stream's residue mod 16 is the one its case chose), outputs 128-byte aligned with
    at least 64 canary bytes after each out_cap."""
    io = np.zeros(len(cs), dtype=pkg.binding.FRAME_IO_DTYPE)
    src = bytearray()
    oo = 0
    for i, c in enumerate(cs):
        src += bytes(-len(src) % 16)
        io[i] = (len(src), len(c.frame), oo, c.cap)
        src += c.frame
        oo = (oo + c.cap + 64 + 127) & ~127
    return io, np.frombuffer(bytes(src), dtype=np.uint8), oo


def _check_tables(got, want, c, blk):
    if want["huf"] is None:
        assert got["huf"] is None, (c, blk)
    else:
        assert got["huf"] is not None and (got["huf"]["max_bits"], got["huf"]["entries"]) == want["huf"], (c, blk, "huf")
    for kind in E.KINDS:
        w, g = want[kind], got[kind]
        if w is None:
            assert g is None, (c, blk, kind)
            continue
        assert g is not None and g["valid"] == 1 and g["is_rle"] == w["is_rle"] and g["log"] == w["log"], (c, blk, kind, g and g["log"])
        bad = [i for i, (a, b) in enumerate(zip(g["entries"], w["entries"])) if a != b]
        assert not bad and len(g["entries"]) == len(w["entries"]), (c, blk, kind, bad[:4])


def _check(pkg, b, cs, io, res, out):
    names = pkg.error_names()
    blk = 0
    for i, c in enumerate(cs):
        r, o = res[i], int(io[i]["out_off"])
        if c.valid:
            assert r["status"] == 0, (c, names[int(r["status"])], int(r["stage"]))
            assert r["out_size"] == len(c.expected) and r["bytes_read"] == len(c.frame), (c, r)
            assert out[o:o + len(c.expected)].tobytes() == c.expected, c
            assert r["has_checksum"] and r["has_calculated_checksum"] and r["calculated_checksum"] == r["checksum_from_data"], c
            for k, (bl, want) in enumerate(zip(c.blocks, c.tables)):
                if want is None:
                    continue
                _check_tables(b.debug_tables(blk + k), want, c, k)
                lits = b.debug_literals(blk + k)
                assert lits == (bl.lits if bl.lit in ("huf", "treeless") else b""), (c, k, "literals")
                seqs = b.debug_sequences(blk + k)
                assert [tuple(int(x) for x in q[:2]) for q in seqs] == [q[:2] for q in bl.seqs], (c, k, "sequences")
        else:
            assert (names[int(r["status"])].replace("B200Z_", ""), int(r["stage"])) == c.err, (c, r)
        end = o + int(io[i]["out_cap"])
        nxt = int(io[i + 1]["out_off"]) if i + 1 < len(cs) else len(out)
        assert (out[end:nxt] == CANARY).all(), (c, "written past out_cap")
        blk += len(c.blocks)


def _run(pkg, ctx, cs):
    import torch
    io, comp, total = _layout(pkg, cs)
    d_out = torch.full((total,), CANARY, dtype=torch.uint8, device="cuda")
    dicts = [pkg.Dictionary.decode_dict(ctx, c.dict_raw) for c in cs if c.dict_raw is not None]
    b = pkg.Batch(ctx, comp, io, dicts=dicts)
    b.run(d_out)
    res = b.finish()
    _check(pkg, b, cs, io, res, d_out.cpu().numpy())
    b.close()


def test_entropy_one_batch(pkg, ctx, crafted, exec_mode, checksummed):
    _run(pkg, ctx, crafted)


def test_entropy_one_frame_per_submission(pkg, ctx, crafted, exec_mode, checksummed):
    for c in crafted:
        _run(pkg, ctx, [c])


def test_entropy_frame_decoder_block_by_block(pkg, ctx, crafted, exec_mode):
    """Treeless, Repeat and dictionary cases one block per submission: the tables reach later blocks through the carry."""
    names = pkg.error_names()
    for c in [c for c in crafted if c.group in ("treeless", "repeat", "dict")]:
        dec = pkg.FrameDecoder(ctx)
        if c.dict_raw is not None:
            dec.add_dict(c.dict_raw)
        if c.valid:
            r = dec.reset(c.frame)
            while not dec.decode_blocks(r, pkg.UPTO_BLOCKS, 1):
                pass
            assert dec.collect() == c.expected, c
            assert dec.bytes_read_from_source() == len(c.frame) and dec.get_checksum_from_data() == dec.get_calculated_checksum()
        else:
            with pytest.raises(pkg.B200ZError) as e:
                r = dec.reset(c.frame)
                while not dec.decode_blocks(r, pkg.UPTO_BLOCKS, 1):
                    pass
            assert (names[e.value.code].replace("B200Z_", ""), e.value.stage) == c.err, (c, e.value)
