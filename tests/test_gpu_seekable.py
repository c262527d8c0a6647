"""Seekable archives on the GPU: compress_seekable's frames are compress_frames' frames for the same pieces, byte for byte, and its
table is the model's (tests/seekable.py) -- at Fastest and LAZY, with and without checksums, with raw-content and formatted
dictionaries, from host and device memory to host and device memory, across groups; the archives decode through decode_all,
decode_all_stream and libzstd.  read_ranges returns exactly the content's slices on these archives and on libzstd-written ones, for
the crafted range sets and 10,000 seeded random ranges, from host and device archives into host and device outputs, leaving the
bytes between slots untouched.  A wrong Decompressed_Size fails only the ranges that touch its frame; a wrong checksum entry is
reported.  Argument checks and launch counts are those of the header."""
import struct

import numpy as np
import pytest
import torch

import datagen
import seekable
from test_seekable_model import libzstd_archive

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def data():
    return {"c2b": datagen.gen_text(1_500_000, 0x5EC1).tobytes(), "silesia": datagen.gen_silesia_mix(1_100_000, 0x5EC2).tobytes()}


@pytest.fixture(scope="module")
def dicts(pkg, ctx, data):
    content = datagen.gen_text(65536, 0x5EC3).tobytes()
    samples = [data["c2b"][i:i + 20000] for i in range(0, 400000, 20000)]
    return {"raw": pkg.Dictionary.raw_content(ctx, 1, content), "formatted": pkg.Dictionary.decode_dict(ctx, pkg.finalize_dict(ctx, content, samples)),
            "content": content}


def pieces_of(plain, fs):
    return [plain[i:i + fs] for i in range(0, len(plain), fs)]


def batch_frames(pkg, ctx, pieces, level, checksum, dict=None, dict_tables=False):
    io = np.zeros(len(pieces), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, p in enumerate(pieces):
        cap = pkg.compress_bound(len(p), dict)
        io[i] = (so, len(p), oo, cap)
        so += len(p); oo += cap
    out = np.zeros(max(oo, 1), dtype=np.uint8)
    src = np.frombuffer(b"".join(pieces), dtype=np.uint8) if so else np.zeros(1, dtype=np.uint8)
    res = pkg.compress_frames(ctx, src, io, out, level, checksum, dict=dict, dict_tables=dict_tables)
    assert (res["status"] == 0).all()
    return [out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(pieces))], res


def model_archive(pkg, ctx, plain, fs, level, checksum, dict=None, dict_tables=False):
    pieces = pieces_of(plain, fs)
    frames, res = batch_frames(pkg, ctx, pieces, level, checksum, dict, dict_tables)
    return seekable.write(frames, [len(p) for p in pieces], [int(r["checksum"]) for r in res] if checksum else None)


def seek(pkg, ctx, plain, fs, level=1, checksum=True, dict=None, dict_tables=False, dev_in=False, dev_out=False):
    inp = torch.frombuffer(bytearray(plain), dtype=torch.uint8).cuda() if dev_in and plain else (plain if not dev_in else torch.zeros(0, dtype=torch.uint8, device="cuda"))
    cap = pkg.seekable_bound(len(plain), fs, checksum, dict)
    out = torch.full((cap,), 0xA5, dtype=torch.uint8, device="cuda") if dev_out else np.full(cap, 0xA5, dtype=np.uint8)
    n = pkg.compress_seekable(ctx, inp, out, fs, level, checksum, dict, dict_tables)
    return (out[:n].cpu().numpy() if dev_out else out[:n]).tobytes()


def decodes(pkg, ctx, archive, plain, dicts=None, forced=None, raw=None):
    out = np.zeros(len(plain) + 64, dtype=np.uint8)
    s, _ = pkg.decode_all(ctx, archive, out, dicts=dicts, forced_dict=forced)
    assert s["status"] == 0 and s["written"] == len(plain) and out[:len(plain)].tobytes() == plain
    got = bytearray()
    r = pkg.decode_all_stream(ctx, archive, got, dicts=dicts, forced_dict=forced)
    assert r["status"] == 0 and bytes(got) == plain
    assert datagen.decompress(archive, len(plain) + 64, raw_dict=raw) == plain


@pytest.mark.parametrize("kind", ["c2b", "silesia"])
@pytest.mark.parametrize("level", [1, 5])
@pytest.mark.parametrize("checksum", [True, False])
def test_frames_and_table_are_the_batch_compressors(pkg, ctx, data, kind, level, checksum):
    plain = data[kind]
    for fs in (200_000, 65536):
        arch = seek(pkg, ctx, plain, fs, level, checksum)
        assert arch == model_archive(pkg, ctx, plain, fs, level, checksum)
        ent, ck = seekable.parse(arch)
        assert ck == checksum and len(ent) == -(-len(plain) // fs)
    decodes(pkg, ctx, arch, plain)


@pytest.mark.parametrize("which", ["raw", "formatted", "formatted_tables"])
@pytest.mark.parametrize("level", [1, 5])
def test_with_dictionaries(pkg, ctx, data, dicts, which, level):
    plain = data["c2b"][:700_000]
    D = dicts["raw" if which == "raw" else "formatted"]
    tables = which == "formatted_tables"
    arch = seek(pkg, ctx, plain, 100_000, level, True, D, tables)
    assert arch == model_archive(pkg, ctx, plain, 100_000, level, True, D, tables)
    if which == "raw":
        decodes(pkg, ctx, arch, plain, forced=D, raw=dicts["content"])
    else:
        out = np.zeros(len(plain) + 64, dtype=np.uint8)
        s, _ = pkg.decode_all(ctx, arch, out, dicts=[D])
        assert s["status"] == 0 and out[:len(plain)].tobytes() == plain
    with pkg.SeekableArchive(ctx, arch) as a:
        kw = {"forced_dict": D} if which == "raw" else {"dicts": [D]}
        assert a.read(123_457, 300_000, **kw) == plain[123_457:423_457]


def test_memory_kinds_and_groups(pkg, ctx, data):
    plain = ((data["c2b"] + data["silesia"]) * 5)[:2600 * 4096 - 1234]   # 2600 frames of 4 KiB: two groups of B200Z_SEEKABLE_GROUP_BLOCKS
    assert -(-len(plain) // 4096) > pkg.binding.SEEKABLE_GROUP_BLOCKS
    want = model_archive(pkg, ctx, plain, 4096, 1, True)
    before = ctx.kernel_launches()
    assert seek(pkg, ctx, plain, 4096) == want
    assert ctx.kernel_launches() - before == 2 * 5 + 1          # per group k_cmatch, k_cenc, k_cxxh64, k_cscan, k_cassemble; one k_cseek
    for dev_in in (False, True):
        for dev_out in (False, True):
            assert seek(pkg, ctx, plain, 4096, dev_in=dev_in, dev_out=dev_out) == want, (dev_in, dev_out)
    decodes(pkg, ctx, want, plain)
    small = data["c2b"][:300_000]
    assert seek(pkg, ctx, small, 1 << 30, level=0, checksum=False, dev_in=True, dev_out=True) == model_archive(pkg, ctx, small, 1 << 30, 0, False)
    want = model_archive(pkg, ctx, small, 131072, 0, False)
    before = ctx.kernel_launches()
    assert seek(pkg, ctx, small, 131072, level=0, checksum=False) == want
    assert ctx.kernel_launches() - before == 3                   # Uncompressed: k_cscan, k_cassemble, k_cseek


def test_empty_input(pkg, ctx):
    for dev in (False, True):
        arch = seek(pkg, ctx, b"", 4096, dev_in=dev, dev_out=dev)
        assert arch == seekable.table([], True)
        with pkg.SeekableArchive(ctx, arch) as a:
            assert a.num_frames == 0 and a.content_size == 0 and a.read(0, 0) == b""


def test_argument_checks(pkg, ctx, data):
    plain = data["c2b"][:10000]
    L = ctx.L
    out = np.zeros(pkg.seekable_bound(len(plain), 4096, True), dtype=np.uint8)
    w = __import__("ctypes").c_size_t()

    def call(fs, cap=out.size, level=1):
        return L.b200z_compress_seekable(ctx.h, plain, len(plain), 0, fs, level, 1, None, out.ctypes.data, cap, 0, __import__("ctypes").byref(w))
    before = ctx.kernel_launches()
    assert call(0) == pkg.binding.ERR_INVALID_ARGUMENT
    assert call((1 << 30) + 1) == pkg.binding.ERR_INVALID_ARGUMENT
    assert call(4096, out.size - 1) == pkg.binding.ERR_INVALID_ARGUMENT
    assert call(4096, level=6) == pkg.binding.ERR_INVALID_ARGUMENT
    assert call(4096, level=3) == 200   # REFERENCE_WOULD_PANIC, as compress_frames
    assert ctx.kernel_launches() == before
    assert call(4096) == 0 and w.value <= out.size
    arch = out[:w.value].tobytes()
    with pkg.SeekableArchive(ctx, arch) as a:
        buf = np.zeros(100, dtype=np.uint8)
        for bad in ([(len(plain) - 5, 6, 0)], [(0, 10, 0), (20, 10, 5)], [(0, 10, 95)]):
            with pytest.raises(pkg.B200ZError) as e:
                a.read_ranges(bad, buf)
            assert e.value.code == pkg.binding.ERR_INVALID_ARGUMENT
    with pytest.raises(pkg.B200ZError) as e:
        pkg.SeekableArchive(ctx, arch[:-1])
    assert e.value.code == pkg.binding.ERR_SEEKABLE_TABLE


def check_reads(pkg, ctx, arch, plain, ranges, end, dev_arch, dev_out):
    src = torch.frombuffer(bytearray(arch), dtype=torch.uint8).cuda() if dev_arch else arch
    with pkg.SeekableArchive(ctx, src) as a:
        assert a.content_size == len(plain)
        out = torch.full((end + 8,), 0xEE, dtype=torch.uint8, device="cuda") if dev_out else np.full(end + 8, 0xEE, dtype=np.uint8)
        res = a.read_ranges(ranges, out)
    got = out.cpu().numpy().tobytes() if dev_out else out.tobytes()
    assert (res["status"] == 0).all(), res[res["status"] != 0][:4]
    mask = np.ones(end + 8, dtype=bool)
    for off, ln, oo in ranges:
        assert got[oo:oo + ln] == plain[off:off + ln], (off, ln, oo)
        mask[oo:oo + ln] = False
    assert (np.frombuffer(got, dtype=np.uint8)[mask] == 0xEE).all(), "a byte outside the slots was written"
    return res


def test_read_ranges(pkg, ctx, data):
    plain = data["c2b"]
    archives = [(seek(pkg, ctx, plain, 131072), plain), (seek(pkg, ctx, plain, 50_000, level=5, checksum=False), plain),
                libzstd_archive(0x5E1, True), libzstd_archive(0x5E2, False)]
    rng = np.random.default_rng(0x5EAD)
    for k, (arch, pl) in enumerate(archives):
        entries, _ = seekable.parse(arch)
        sets = list(seekable.crafted_ranges(entries).values())
        sets.append(seekable.random_ranges(len(pl), 10_000, rng, 1, 4096)[0])
        for i, rs in enumerate(sets):
            end = max(oo + ln for _, ln, oo in rs) + 1
            for dev_arch, dev_out in ((False, False), (True, True), (True, False), (False, True)):
                res = check_reads(pkg, ctx, arch, pl, rs, end, dev_arch, dev_out)
            assert [int(x) for x in res["frames"]] == [len(t) for t in seekable.plan(entries, rs)[3]]


def test_device_archive_to_host(pkg, ctx, data):
    """The common Python call: a device archive read into host memory, on a fresh context (nothing sized by an earlier call), then
    after a host-archive read that leaves a smaller pinned buffer behind."""
    plain = data["silesia"]
    arch = seek(pkg, ctx, plain, 65536)
    dev = torch.frombuffer(bytearray(arch), dtype=torch.uint8).cuda()
    fresh = pkg.Context(0)
    try:
        with pkg.SeekableArchive(fresh, dev) as a:
            assert a.read(70_000, 500_000) == plain[70_000:570_000]
        with pkg.SeekableArchive(fresh, arch) as a:
            assert a.read(5, 100) == plain[5:105]
        with pkg.SeekableArchive(fresh, dev) as a:
            assert a.read(1, len(plain) - 1) == plain[1:]
    finally:
        fresh.close()


def test_staging_follows_the_input(pkg, ctx, data):
    """A small input with a large frame_size holds the staging of its own blocks, not of a full frame's (8192 blocks, ~7.4 GB)."""
    small = data["c2b"][:300_000]
    fresh = pkg.Context(0)
    try:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        cap = pkg.seekable_bound(len(small), 1 << 30, True)
        out = np.zeros(cap, dtype=np.uint8)
        n = pkg.compress_seekable(fresh, small, out, 1 << 30)
        torch.cuda.synchronize()
        held = free0 - torch.cuda.mem_get_info()[0]
        assert out[:n].tobytes() == model_archive(pkg, ctx, small, 1 << 30, 1, True)
        assert held < 256 << 20, held
    finally:
        fresh.close()


def test_wrong_entries(pkg, ctx, data):
    plain = data["silesia"][:1_000_000]
    arch = bytearray(seek(pkg, ctx, plain, 100_000))
    entries, _ = seekable.parse(bytes(arch))
    at = len(arch) - (17 + 12 * len(entries))
    k = 4
    struct.pack_into("<I", arch, at + 8 + 12 * k + 4, entries[k][3] - 1)             # Decompressed_Size one short
    view = plain[:entries[k][2]] + plain[entries[k][2]:entries[k][2] + entries[k][3] - 1] + plain[entries[k][2] + entries[k][3]:]
    ranges = [(0, 5000, 0), (entries[k][2] + 10, 100, 6000), (entries[k][2] - 50, 100, 7000), (entries[k + 1][2] + 7, 2000, 8000),
              (0, len(view), 20000)]
    with pkg.SeekableArchive(ctx, bytes(arch)) as a:
        out = np.zeros(20000 + len(view), dtype=np.uint8)
        res = a.read_ranges(ranges, out)
    assert [int(s) for s in res["status"]] == [0, 241, 241, 0, 241]
    assert [int(f) for f in res["error_frame"]] == [-1, k, k, -1, k]
    assert out[:5000].tobytes() == view[:5000] and out[8000:10000].tobytes() == view[entries[k + 1][2] + 7:entries[k + 1][2] + 2007]
    arch = bytearray(seek(pkg, ctx, plain, 100_000))
    struct.pack_into("<I", arch, at + 8 + 12 * k + 8, entries[k][4] ^ 1)              # checksum entry flipped
    ctx.set_flags(pkg.binding.FLAG_CHECKSUM)
    try:
        with pkg.SeekableArchive(ctx, bytes(arch)) as a:
            out = np.zeros(20000 + len(plain) + 8, dtype=np.uint8)
            res = a.read_ranges([(0, 5000, 0), (entries[k][2] + 10, 100, 6000), (0, len(plain), 20000)], out)
    finally:
        ctx.set_flags(0)
    assert [int(s) for s in res["status"]] == [0, 0, 0]
    assert [int(m) for m in res["checksum_mismatches"]] == [0, 1, 1]
    assert out[20000:20000 + len(plain)].tobytes() == plain


def test_read_launch_counts(pkg, ctx, data):
    plain = data["c2b"][:800_000]
    arch = seek(pkg, ctx, plain, 131072)
    entries, _ = seekable.parse(arch)
    io = np.array([(e[0], e[1], e[2], e[3]) for e in entries], dtype=pkg.binding.FRAME_IO_DTYPE)
    b = pkg.Batch(ctx, arch, io)                                  # a host archive: no k_walk in either
    out = torch.zeros(len(plain) + 16, dtype=torch.uint8, device="cuda")
    b.run(out)
    b.finish()
    per_pass = b.info()["launches_per_run"]
    b.close()
    with pkg.SeekableArchive(ctx, arch) as a:
        for ranges, gathers in (([(0, len(plain), 0)], 0), ([(1, len(plain) - 1, 0)], 1), ([(5, 0, 0)], None)):
            before = ctx.kernel_launches()
            assert (a.read_ranges(ranges, out)["status"] == 0).all()
            assert ctx.kernel_launches() - before == (0 if gathers is None else per_pass + gathers)
        fr = a.frames
    assert [tuple(int(x) for x in r)[:4] for r in fr] == [e[:4] for e in entries]
    assert [int(x) for x in fr["checksum"]] == [e[4] for e in entries]
