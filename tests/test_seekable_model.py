"""Seekable archives without a GPU: the model (tests/seekable.py) against libzstd and the oracle on archives of libzstd frames, the
library's read plan (b200z_debug_seekable_plan) against the model's on crafted and seeded random range sets, each corrupt-table
rule and each range check with its code, and b200z_seekable_bound."""
import ctypes as C
import struct

import numpy as np
import pytest

import datagen
import seekable

ZSTD_c_compressionLevel, ZSTD_c_checksumFlag, ZSTD_c_contentSizeFlag = 100, 201, 200


def libzstd_frame(data, level=3):
    """A libzstd frame without Frame_Content_Size (as a streaming writer leaves it), with its checksum."""
    z = datagen.zstd()
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    cap = z.ZSTD_compressBound(len(a))
    dst = np.empty(cap, dtype=np.uint8)
    cctx = z.ZSTD_createCCtx()
    try:
        z.ZSTD_CCtx_setParameter(cctx, ZSTD_c_compressionLevel, level)
        z.ZSTD_CCtx_setParameter(cctx, ZSTD_c_checksumFlag, 1)
        z.ZSTD_CCtx_setParameter(cctx, ZSTD_c_contentSizeFlag, 0)
        n = z.ZSTD_compress2(cctx, dst.ctypes.data, cap, a.ctypes.data if len(a) else None, len(a))
    finally:
        z.ZSTD_freeCCtx(cctx)
    assert not z.ZSTD_isError(n)
    return dst[:n].tobytes()


def libzstd_archive(seed, checksum=True):
    """(archive, plaintext): multi-block libzstd frames of C2b-shaped text and Silesia-shaped data, an empty frame and a skippable
    frame with a 0-size entry in between."""
    rng = np.random.default_rng(seed)
    sizes = [300000, 1, 131072, 0, 262145, 77777, 5000]
    pieces, frames = [], []
    for i, n in enumerate(sizes):
        d = (datagen.gen_text if i % 2 == 0 else datagen.gen_silesia_mix)(n, seed + i).tobytes()[:n] if n else b""
        pieces.append(d)
        frames.append(libzstd_frame(d))
    skip = struct.pack("<II", 0x184D2A50 + int(rng.integers(0, 16)), 7) + b"skipped"
    frames.insert(3, skip)
    pieces.insert(3, b"")
    sums = [datagen_xxh64_low(p) for p in pieces]
    sums[3] = 0
    archive = seekable.write(frames, [len(p) for p in pieces], sums if checksum else None)
    return archive, b"".join(pieces)


def datagen_xxh64_low(data):
    from oracle import oracle
    return oracle.xxh64(data) & 0xFFFFFFFF


@pytest.fixture(scope="module")
def archives():
    return [libzstd_archive(0x5E1, True), libzstd_archive(0x5E2, False)]


def test_model_archives_decode_with_libzstd_and_the_oracle(archives, oracle):
    for archive, plain in archives:
        assert datagen.decompress(archive, len(plain) + 16) == plain
        d = oracle.FrameDecoder()
        assert d.decode_all(archive, len(plain) + 16) == plain
        entries, _ = seekable.parse(archive)
        assert sum(e[3] for e in entries) == len(plain)


def test_model_table_round_trip():
    for ck in (False, True):
        ent = [(10, 20, 0xDEADBEEF), (0, 0, 0), (5, 1 << 31, 7)]
        arch = b"x" * 15 + seekable.table(ent, ck)
        got, flag = seekable.parse(arch)
        assert flag == ck
        assert [(c, d) for _, c, _, d, _ in got] == [(c, d) for c, d, _ in ent]
        assert len(seekable.table(ent, ck)) == 17 + len(ent) * (12 if ck else 8)


def _plan(pkg, archive, ranges):
    fr, pc, scr = pkg.seekable_plan(archive, ranges)
    return ([(int(a), int(b), int(c)) for a, b, c in fr], [tuple(int(x) for x in p) for p in pc], scr)


def test_plan_matches_the_model_on_crafted_ranges(pkg, archives):
    for archive, plain in archives:
        entries, _ = seekable.parse(archive)
        for name, rs in seekable.crafted_ranges(entries).items():
            mf, mp, ms, _ = seekable.plan(entries, rs)
            assert _plan(pkg, archive, rs) == (mf, mp, ms), name
            out = seekable.execute(plain, entries, rs, max(oo + ln for _, ln, oo in rs) + 1)
            for off, ln, oo in rs:
                assert out[oo:oo + ln] == plain[off:off + ln], name


def test_plan_rules_on_a_frame_inside_two_ranges(pkg, archives):
    archive, _ = archives[0]
    entries, _ = seekable.parse(archive)
    rs = seekable.crafted_ranges(entries)["two_contain"]
    frames, pieces, scratch = _plan(pkg, archive, rs)
    f = [e for e in entries if e[3]][1]
    idx = entries.index(f)
    assert (idx, rs[0][2] + f[2] - rs[0][0], 0) in frames          # in place for the first range that holds it wholly
    assert all(p[3] == 0 for p in pieces if p[4] == 2)              # the third range copies it from the first range's slot
    assert scratch > 0


def test_plan_matches_the_model_on_random_ranges(pkg, archives):
    rng = np.random.default_rng(0x5EE)
    for archive, plain in archives:
        entries, _ = seekable.parse(archive)
        content = len(plain)
        for _ in range(20):
            n = int(rng.integers(1, 40))
            rs, end = seekable.random_ranges(content, n, rng, 0, int(rng.choice([16, 4096, 300000])))
            perm = rng.permutation(n)
            rs = [rs[i] for i in perm]                              # slots need not follow call order
            mf, mp, ms, _ = seekable.plan(entries, rs)
            assert _plan(pkg, archive, rs) == (mf, mp, ms)
            out = seekable.execute(plain, entries, rs, end)
            for off, ln, oo in rs:
                assert out[oo:oo + ln] == plain[off:off + ln]


def _corrupt(archive, n_entries, ck):
    esz = 12 if ck else 8
    tb = 17 + n_entries * esz
    at = len(archive) - tb
    out = {}
    b = bytearray(archive); b[-1] ^= 0xFF; out["footer_magic"] = bytes(b)
    b = bytearray(archive); b[-5] |= 0x04; out["reserved_bits"] = bytes(b)
    b = bytearray(archive); struct.pack_into("<I", b, at + 4, n_entries * esz + 10); out["frame_size"] = bytes(b)
    b = bytearray(archive); struct.pack_into("<I", b, len(b) - 9, 1 << 28); out["n_too_large"] = bytes(b)
    b = bytearray(archive); struct.pack_into("<I", b, at + 8, struct.unpack_from("<I", b, at + 8)[0] + 1); out["sum"] = bytes(b)
    out["truncated"] = archive[:len(archive) - 5]
    b = bytearray(archive); b[at] ^= 1; out["skippable_magic"] = bytes(b)
    out["tiny"] = archive[-12:]
    return out


def test_corrupt_tables_fail_with_the_table_code(pkg, archives):
    for archive, _ in archives:
        entries, ck = seekable.parse(archive)
        for name, bad in _corrupt(archive, len(entries), ck).items():
            with pytest.raises(seekable.TableError):
                seekable.parse(bad)
            with pytest.raises(pkg.B200ZError) as e:
                pkg.seekable_plan(bad, [(0, 1, 0)])
            assert e.value.code == pkg.binding.ERR_SEEKABLE_TABLE, name
    assert pkg.lib().b200z_error_name(240) == b"ERR_SEEKABLE_TABLE"
    assert pkg.lib().b200z_error_name(241) == b"ERR_SEEKABLE_FRAME_SIZE"
    assert pkg.error_names()[240] == "B200Z_ERR_SEEKABLE_TABLE" and pkg.error_names()[241] == "B200Z_ERR_SEEKABLE_FRAME_SIZE"


def test_range_checks(pkg, archives):
    archive, plain = archives[0]
    n = len(plain)
    for bad in ([(n - 10, 11, 0)], [(n + 1, 0, 0)], [(0, 100, 0), (500, 100, 99)], [(0, 10, 5), (20, 10, 0)]):
        with pytest.raises(seekable.RangeError):
            seekable.plan(seekable.parse(archive)[0], bad)
        with pytest.raises(pkg.B200ZError) as e:
            pkg.seekable_plan(archive, bad)
        assert e.value.code == pkg.binding.ERR_INVALID_ARGUMENT
    # touching slots, empty ranges anywhere and ranges overlapping in the content are fine
    pkg.seekable_plan(archive, [(0, 100, 0), (50, 100, 100), (n, 0, 0), (3, 0, 7)])


def test_empty_archive_plan(pkg):
    arch = seekable.table([], True)
    fr, pc, scr = pkg.seekable_plan(arch, [(0, 0, 0)])
    assert len(fr) == 0 and len(pc) == 0 and scr == 0


def test_seekable_bound(pkg):
    cb = pkg.compress_bound
    assert pkg.seekable_bound(0, 4096, True) == 17
    assert pkg.seekable_bound(10000, 4096, True) == 2 * cb(4096) + cb(10000 - 8192) + 17 + 3 * 12
    assert pkg.seekable_bound(8192, 4096, False) == 2 * cb(4096) + 17 + 2 * 8
    assert pkg.seekable_bound(100, 0, True) == 0
    assert pkg.seekable_bound(100, (1 << 30) + 1, True) == 0
    assert pkg.seekable_bound(100, 1 << 30, True) == cb(100) + 29
