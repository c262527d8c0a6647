"""The zstd dictionary writer of b200z_dict_finalize, on the host (b200z_debug_dict_from_counts, no GPU): dictionaries from crafted
statistics must load in the oracle (ruzstd's Dictionary::decode_dict) and in libzstd, and work both ways: libzstd compresses with
them at levels 1 and 3 and the oracle decodes those frames by ID.  Also: the ID rule against libzstd's ZDICT_finalizeDictionary,
trimming to dict_cap, the header bound and the argument checks."""
import ctypes as C
import struct

import numpy as np
import pytest

import datagen

LIT, LL, ML, OF = 0, 256, 256 + 36, 256 + 36 + 53
NBINS = OF + 32


@pytest.fixture(scope="module")
def content():
    return datagen.gen_text(30000, 0xD1C7).tobytes()


def crafted(content_len):
    """(name, counts[377]) for the cases the writer must handle."""
    rng = np.random.default_rng(7)
    z = np.zeros(NBINS, dtype=np.uint64)
    out = [("flat", z.copy() + 1000), ("no samples", z.copy())]
    one = z.copy()
    one[LIT + ord("e")] = 10**9
    one[LL + 0] = one[ML + 2] = one[OF + 10] = 10**9
    out.append(("one dominant symbol", one))
    but = z.copy() + 5000
    but[LIT + 7] = 1
    but[LL + 35] = but[ML + 52] = but[OF + 3] = 1
    out.append(("every symbol equal but one", but))
    ofmax = (content_len + 131072).bit_length() - 1
    of = rng.integers(1, 1000, NBINS).astype(np.uint64)
    of[OF:OF + 32] = 0
    of[OF + ofmax] = 10**6
    out.append(("OF codes up to the content's maximum", of))
    wide = rng.integers(0, 2**40, NBINS).astype(np.uint64)   # totals far above 2^32
    out.append(("large counts", wide))
    skew = (2.0 ** rng.uniform(0, 30, NBINS)).astype(np.uint64)
    skew[OF + 31] = 12345                                    # an OF code beyond the content's maximum, zeros before it
    out.append(("skewed", skew))
    return out


def parse(d):
    """The ID of a dictionary (after checking its magic number)."""
    assert d[:4] == bytes.fromhex("37a430ec")
    return struct.unpack_from("<I", d, 4)[0]


def oracle_round_trip(oracle, d, frame, data):
    dec = oracle.FrameDecoder()
    dec.add_dict(d)
    r = dec.reset(frame)
    dec.decode_blocks(r)
    assert dec.collect() == data


def zdict_finalize(content, samples, dict_id=0, cap=None):
    z = datagen.zstd()
    z.ZDICT_finalizeDictionary.restype = C.c_size_t

    class Params(C.Structure):
        _fields_ = [("compressionLevel", C.c_int), ("notificationLevel", C.c_uint), ("dictID", C.c_uint)]
    z.ZDICT_finalizeDictionary.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint, Params]
    z.ZDICT_isError.restype = C.c_uint
    z.ZDICT_isError.argtypes = [C.c_size_t]
    z.ZDICT_getDictID.restype = C.c_uint
    z.ZDICT_getDictID.argtypes = [C.c_void_p, C.c_size_t]
    cap = cap or len(content) + 4096
    out = np.zeros(cap, dtype=np.uint8)
    buf = np.frombuffer(b"".join(samples), dtype=np.uint8)
    sizes = np.array([len(s) for s in samples], dtype=np.uintp)
    n = z.ZDICT_finalizeDictionary(out.ctypes.data, cap, content, len(content), buf.ctypes.data, sizes.ctypes.data, len(samples),
                                   Params(3, 0, dict_id))
    assert not z.ZDICT_isError(n)
    return out[:n].tobytes(), z.ZDICT_getDictID(out.ctypes.data, n)


@pytest.mark.parametrize("case", range(7))
def test_crafted_counts_load_everywhere(pkg, oracle, content, case):
    name, counts = crafted(len(content))[case]
    d = pkg.dict_from_counts(counts, content)
    assert parse(d) >= 32768
    assert d.endswith(content) and len(d) - len(content) <= pkg.binding.DICT_HEADER_MAX, name
    assert d[len(d) - len(content) - 12:len(d) - len(content)] == struct.pack("<III", 1, 4, 8)
    data = datagen.gen_text(40000, 11).tobytes() + content[5000:9000] + bytes(range(256)) * 4
    for level in (1, 3):
        f = datagen.compress(data, level=level, raw_dict=d)
        assert f[4] & 3, "libzstd wrote no dictionary ID: it did not load the dictionary as a formatted one"
        assert datagen.decompress(f, len(data), raw_dict=d) == data
        oracle_round_trip(oracle, d, f, data)
    assert pkg.dict_from_counts(counts, content) == d   # deterministic


def test_oracle_reads_the_same_content(pkg, oracle, content):
    """A frame whose first sequence copies from the content's first bytes decodes only if the oracle found the content where the
    writer put it (libzstd level 3 finds those matches)."""
    d = pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64) + 3, content)
    data = content[:3000] + content[-3000:]
    f = datagen.compress(data, level=3, raw_dict=d)
    assert len(f) < 600
    oracle_round_trip(oracle, d, f, data)


def test_derived_id_is_libzstds(pkg, content):
    samples = [datagen.gen_text(2000, 100 + i).tobytes() for i in range(50)]
    for c in (content, content[:8], content[:1000]):
        zd, zid = zdict_finalize(c, samples)
        d = pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64), c)
        assert parse(d) == zid == parse(zd), len(c)
        assert pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64), c, dict_id=77)[4:8] == struct.pack("<I", 77)
    d = pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64), content, dict_id=(1 << 31) - 1)
    assert parse(d) == (1 << 31) - 1


def test_trimming_keeps_the_tail(pkg, content):
    counts = crafted(len(content))[3][1]
    full = pkg.dict_from_counts(counts, content, dict_id=5)
    h = len(full) - len(content)
    for cap in (len(full), len(full) - 1, 1000, pkg.binding.DICT_HEADER_MAX + 8):
        d = pkg.dict_from_counts(counts, content, dict_id=5, dict_cap=cap)
        keep = min(len(content), cap - h)
        assert len(d) == h + keep and d[:h] == full[:h] and d[h:] == content[len(content) - keep:]
    # a derived ID is the one of the content written
    d = pkg.dict_from_counts(counts, content, dict_cap=2000)
    assert parse(d) == parse(pkg.dict_from_counts(counts, d[len(d) - (2000 - h):]))


def test_argument_checks(pkg, content):
    bad = {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_INVALID_ARGUMENT"]
    z = np.zeros(NBINS, dtype=np.uint64)
    for kw in ({"content": content[:7]}, {"dict_id": 1 << 31}, {"dict_id": 0xFFFFFFFF}, {"dict_cap": pkg.binding.DICT_HEADER_MAX + 7}):
        args = {"content": content, "dict_id": 0, "dict_cap": None}
        args.update(kw)
        with pytest.raises(pkg.B200ZError) as e:
            pkg.dict_from_counts(z, args["content"], dict_id=args["dict_id"], dict_cap=args["dict_cap"])
        assert e.value.code == bad, kw
    assert len(pkg.dict_from_counts(z, content[:8], dict_cap=pkg.binding.DICT_HEADER_MAX + 8)) <= pkg.binding.DICT_HEADER_MAX + 8


def test_reserved_ids_are_accepted_by_libzstd_and_the_oracle(pkg, oracle, content):
    """Why IDs >= 2^31 are refused by the writer rather than by the readers: the format reserves them, but libzstd and ruzstd load
    and use such a dictionary like any other."""
    d = pkg.dict_from_counts(np.zeros(NBINS, dtype=np.uint64), content, dict_id=7)
    d = d[:4] + struct.pack("<I", 0x80000001) + d[8:]
    data = content[100:4000] * 3
    f = datagen.compress(data, level=3, raw_dict=d)
    assert datagen.decompress(f, len(data), raw_dict=d) == data
    oracle_round_trip(oracle, d, f, data)
