"""The batch compressor with a formatted dictionary's entropy tables (B200Z_FLAG_DICT_TABLES, dict_tables=True), on the GPU: every
frame decodes with libzstd, the oracle (by ID), decode_frames in both execution modes, decode_all and FrameDecoder.add_dict, carries
the ID and checksum, stays within compress_bound_dict and the 128 KiB window; Treeless / Repeat appear in first blocks only; without
the flag, or with raw content, the output is unchanged; no extra launch; the held-out ratio improves."""
import struct

import numpy as np
import pytest

import datagen
from conftest import read_golden
from test_compress_dict import batch_decode, compress_many, header_dict_id, oracle_trace
from test_dict_format_host import crafted, zdict_finalize

pytestmark = pytest.mark.gpu
WINDOW = 131072


@pytest.fixture(scope="module")
def c5():
    fs = datagen.config_c5(nframes=4000, cache=False)
    plain = fs.plain.tobytes()
    return [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)], fs.raw_dict.tobytes()


@pytest.fixture(scope="module")
def finalized(pkg, ctx, c5):
    pieces, content = c5
    return pkg.finalize_dict(ctx, content, pieces[:2000])


def block_modes(f):
    """[(literals type, (LL, OF, ML) modes or None)] of each Compressed block of a frame, None for the other blocks."""
    fhd = f[4]
    did = (0, 1, 2, 4)[fhd & 3]
    fcs = (1 if fhd & 0x20 else 0, 2, 4, 8)[fhd >> 6]
    p = 4 + 1 + (0 if fhd & 0x20 else 1) + did + fcs
    out = []
    while True:
        h = int.from_bytes(f[p:p + 3], "little")
        last, bt, size = h & 1, (h >> 1) & 3, h >> 3
        p += 3
        if bt != 2:
            out.append(None)
            p += 1 if bt == 1 else size
        else:
            b = f[p:p + size]
            lt, sf = b[0] & 3, (b[0] >> 2) & 3
            if lt < 2:
                hs = 1 if sf in (0, 2) else 2 if sf == 1 else 3
                v = int.from_bytes(b[:hs], "little")
                regen = v >> 3 if sf in (0, 2) else v >> 4
                q = hs + (regen if lt == 0 else 1)
            else:
                hs = 3 if sf < 2 else 4 if sf == 2 else 5
                v = int.from_bytes(b[:hs], "little")
                bits = 10 if sf < 2 else 14 if sf == 2 else 18
                q = hs + ((v >> (4 + bits)) & ((1 << bits) - 1))
            n = b[q]
            nseq, q = (n, q + 1) if n < 128 else ((((n - 128) << 8) + b[q + 1], q + 2) if n < 255 else (b[q + 1] + (b[q + 2] << 8) + 0x7F00, q + 3))
            modes = None if nseq == 0 else ((b[q] >> 6) & 3, (b[q] >> 4) & 3, (b[q] >> 2) & 3)
            out.append((lt, modes))
            p += size
        if last:
            return out


def uses_tables(m):
    return m is not None and (m[0] == 3 or (m[1] is not None and 3 in m[1]))


def test_round_trips_with_tables(pkg, ctx, oracle, c5, finalized, monkeypatch):
    pieces, content = c5
    d = finalized
    did = struct.unpack_from("<I", d, 4)[0]
    D = pkg.Dictionary.decode_dict(ctx, d)
    extra = [bytes(datagen.gen_text(n, 31 + n)) if n else b"" for n in (0, 1, 131071, 131073)]
    extra += [b"\x2a" * 5000, np.random.default_rng(5).integers(0, 256, 100000, dtype=np.uint8).tobytes(), bytes(datagen.gen_text(8 << 20, 32))]
    datas = pieces[2000:] + extra
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, x in enumerate(datas):
        cap = pkg.compress_bound(len(x), D)
        io[i] = (so, len(x), oo, cap)
        so += len(x)
        oo += cap
    out = np.zeros(oo, dtype=np.uint8)
    res = pkg.compress_frames(ctx, np.frombuffer(b"".join(datas), dtype=np.uint8), io, out, dict=D, dict_tables=True)
    frames = [out[int(io[i]["dst_off"]):int(io[i]["dst_off"] + res[i]["dst_size"])].tobytes() for i in range(len(datas))]
    first = later = 0
    for x, f, r in zip(datas, frames, res):
        assert r["status"] == 0
        assert header_dict_id(f) == (True, did) and len(f) <= pkg.compress_bound(len(x), D)
        assert r["checksum"] == pkg.xxh64(x) & 0xFFFFFFFF and struct.unpack("<I", f[-4:])[0] == r["checksum"]
        assert datagen.decompress(f, len(x), raw_dict=d) == x
        got, _, max_off = oracle_trace(oracle, f, formatted=d)   # by ID; checks the 128 KiB window
        assert got == x and max_off <= WINDOW
        m = block_modes(f)
        first += uses_tables(m[0])
        later += sum(uses_tables(b) for b in m[1:])
    print(f"first blocks coded with the dictionary's tables: {first} of {len(frames)}")
    assert first > 0 and later == 0
    for mode in ("warp", "cta"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, datas, frames, dicts=[D])
    monkeypatch.delenv("B200Z_EXEC_MODE")
    cat = b"".join(frames)
    buf = np.zeros(sum(len(x) for x in datas) + 64, dtype=np.uint8)
    summary, _ = pkg.decode_all(ctx, cat, buf, dicts=[D])
    assert summary["status"] == 0 and buf[:summary["written"]].tobytes() == b"".join(datas)
    fd = pkg.FrameDecoder(ctx)
    fd.add_dict(d)
    for x, f in zip(datas[::37], frames[::37]):
        r = fd.reset(f)
        fd.decode_blocks(r, pkg.ALL)
        assert fd.collect() == x
    assert pkg.compress_to_vec(ctx, datas[5], dict=D, dict_tables=True) == frames[5]


def test_unchanged_without_the_flag(pkg, ctx, c5, finalized):
    """The flag changes nothing without a formatted dictionary, and nothing is left set after a dict_tables=True call."""
    pieces, content = c5
    datas = pieces[2000:2300] + [bytes(datagen.gen_text(300000, 3))]
    R = pkg.Dictionary.raw_content(ctx, 1, content)
    assert compress_many(pkg, ctx, datas, dict=R)[0] == [pkg.compress_to_vec(ctx, x, dict=R, dict_tables=True) for x in datas]
    assert compress_many(pkg, ctx, datas)[0] == [pkg.compress_to_vec(ctx, x, dict_tables=True) for x in datas]
    for raw in (read_golden("dict_tests", "dictionary"), finalized):
        D = pkg.Dictionary.decode_dict(ctx, raw)
        plain, _ = compress_many(pkg, ctx, datas, dict=D)
        pkg.compress_to_vec(ctx, datas[0], dict=D, dict_tables=True)
        assert compress_many(pkg, ctx, datas, dict=D)[0] == plain
        assert pkg.lib().b200z_ctx_flags(ctx.h) & pkg.binding.FLAG_DICT_TABLES == 0


def test_launches_and_rejections(pkg, ctx, c5, finalized):
    pieces, _ = c5
    D = pkg.Dictionary.decode_dict(ctx, finalized)
    L = pkg.lib()
    bad = {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_INVALID_ARGUMENT"]
    src = np.frombuffer(pieces[0], dtype=np.uint8)
    out = np.zeros(pkg.compress_bound(src.size, D), dtype=np.uint8)
    res = np.zeros(1, dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    io = np.array([(0, src.size, 0, out.size - 1)], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    before = ctx.kernel_launches()
    L.b200z_ctx_set_flags(ctx.h, pkg.binding.FLAG_DICT_TABLES)
    try:
        assert L.b200z_compress_frames_batch_dict(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, 1, 1, 1, D.h, out.ctypes.data, out.size, 0,
                                                  res.ctypes.data) == bad
    finally:
        L.b200z_ctx_set_flags(ctx.h, 0)
    assert ctx.kernel_launches() == before
    compress_many_tables(pkg, ctx, pieces[:300], D)
    assert ctx.kernel_launches() - before == 5   # k_cdict once, then the four stages; the tables cost no launch
    compress_many_tables(pkg, ctx, pieces[:300], D)
    assert ctx.kernel_launches() - before == 9


def compress_many_tables(pkg, ctx, datas, D, checksum=True):
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, x in enumerate(datas):
        cap = pkg.compress_bound(len(x), D)
        io[i] = (so, len(x), oo, cap)
        so += len(x)
        oo += cap
    out = np.zeros(oo, dtype=np.uint8)
    res = pkg.compress_frames(ctx, np.frombuffer(b"".join(datas), dtype=np.uint8), io, out, checksum=checksum, dict=D, dict_tables=True)
    assert (res["status"] == 0).all()
    return [out[int(io[i]["dst_off"]):int(io[i]["dst_off"] + res[i]["dst_size"])].tobytes() for i in range(len(datas))]


def test_held_out_ratio(pkg, ctx, c5, finalized):
    """On the 2,000 held-out C5 frames, the dictionary's tables must beat the same dictionary without them, in aggregate."""
    pieces, content = c5
    held = pieces[2000:]
    D = pkg.Dictionary.decode_dict(ctx, finalized)
    total = sum(len(p) for p in held)
    without = sum(len(f) for f in compress_many(pkg, ctx, held, dict=D, checksum=False)[0])
    with_tables = sum(len(f) for f in compress_many_tables(pkg, ctx, held, D, checksum=False))
    zd, _ = zdict_finalize(content, pieces[:2000])
    z1 = total / sum(len(datagen.compress(p, level=1, raw_dict=zd)) for p in held)
    z3 = total / sum(len(datagen.compress(p, level=3, raw_dict=zd)) for p in held)
    print(f"held-out C5 ratio with the finalized dictionary: tables {total / with_tables:.3f}, without {total / without:.3f}; "
          f"libzstd with ZDICT_finalizeDictionary's: level 1 {z1:.3f}, level 3 {z3:.3f}")
    assert with_tables < without


def test_crafted_dictionaries_in_this_library(pkg, ctx, oracle):
    """Dictionaries from crafted counts load with Dictionary.decode_dict: libzstd frames made with them decode here, and this
    compressor's frames with their tables decode with libzstd and the oracle."""
    content = datagen.gen_text(30000, 0xD1C7).tobytes()
    data = datagen.gen_text(40000, 11).tobytes() + content[5000:9000] + bytes(range(256)) * 4
    pieces = [data[i:i + 3000] for i in range(0, len(data), 3000)]
    for name, counts in crafted(len(content)):
        d = pkg.dict_from_counts(counts, content)
        D = pkg.Dictionary.decode_dict(ctx, d)
        assert D.id == struct.unpack_from("<I", d, 4)[0] and D.offset_hist == [1, 4, 8], name
        for level in (1, 3):
            batch_decode(pkg, ctx, pieces, [datagen.compress(p, level=level, raw_dict=d) for p in pieces], dicts=[D])
        for p, f in zip(pieces, compress_many_tables(pkg, ctx, pieces, D)):
            assert datagen.decompress(f, len(p), raw_dict=d) == p, name
            assert oracle.decode_frame(f, dict_raw=d)[0] == p, name
