"""Seekable archives larger than memory.  compress_seekable_stream writes, from a reader to a writer, exactly the archive
compress_seekable writes for the whole input -- at every level, with and without checksums, with raw-content and formatted
dictionaries, at several chunk sizes, frame sizes (one byte up to past the chunk) and input lengths, from sources that return seeded
random short reads -- holding memory, by the library's own count, that does not grow with the source beyond the seek table.  A failing source or drain gives
ERR_SEEKABLE_IO and leaves the context as it was.  SeekableArchive.from_source reads an archive through a positional-read callback:
the same bytes and result rows as the in-memory archive, the same launches, and only the footer, the table (its header first) and
the touched frames' bytes asked for, one call per run of adjacent touched frames."""
import gc
import io
import random
import struct

import numpy as np
import pytest
import torch

import datagen
import seekable

pytestmark = pytest.mark.gpu

ENV = "B200Z_PIPELINE_CHUNK_BYTES"
DEFAULT = 64 << 20
CHUNKS = [131072, 1 << 20, DEFAULT]
FRAME_SIZES = [1, 4103, 131072, 3 * 131072 + 5, (1 << 20) + 12345]   # the last one is larger than every chunk but the default


@pytest.fixture(scope="module")
def data():
    return {"c2b": datagen.gen_text(1_300_000, 0x5E51).tobytes(), "silesia": datagen.gen_silesia_mix(1_300_000, 0x5E52).tobytes()}


class Source:
    """A reader that hands out seeded random short reads (or whole ones), optionally raising at read call `fail_at`."""

    def __init__(self, data, seed=None, fail_at=None):
        self.b, self.pos, self.calls, self.fail_at = data, 0, 0, fail_at
        self.rng = random.Random(seed) if seed is not None else None

    def read(self, n):
        self.calls += 1
        if self.fail_at is not None and self.calls >= self.fail_at:
            raise IOError("source failed")
        if self.rng is not None:
            n = min(n, self.rng.choice([1, 3, 17, 4096, 65536, 1 << 20]))
        out = self.b[self.pos:self.pos + n]
        self.pos += len(out)
        return out


class Drain:
    """A writer that raises (or returns 0, `full`) at write call `fail_at`."""

    def __init__(self, fail_at=None, full=False):
        self.out, self.calls, self.fail_at, self.full = bytearray(), 0, fail_at, full

    def write(self, b):
        self.calls += 1
        if self.fail_at is not None and self.calls >= self.fail_at:
            if self.full:
                return 0
            raise IOError("drain failed")
        self.out += b
        return len(b)


def set_chunk(monkeypatch, chunk):
    monkeypatch.setenv(ENV, str(chunk))


def stream(pkg, ctx, plain, fs, level=1, checksum=True, seed=1, **kw):
    out = bytearray()
    r = pkg.compress_seekable_stream(ctx, Source(plain, seed), out, fs, level, checksum, **kw)
    assert r["read"] == len(plain) and r["written"] == len(out) and r["frames"] == -(-len(plain) // fs)
    return bytes(out), r


def groups_of(n, fs, chunk):
    """the groups the header's rule gives: the most whole frames within the chunk and B200Z_SEEKABLE_GROUP_BLOCKS blocks, at least one"""
    per = max(1, min(chunk // fs, 2048 // max(1, -(-fs // 131072))))
    return -(-n // (per * fs))


def lengths(fs):
    m = max(1, min(5000, 1_200_000 // fs))
    return [0, 1, m * fs - 1, m * fs, m * fs + 1]


@pytest.mark.parametrize("kind", ["c2b", "silesia"])
@pytest.mark.parametrize("level", [0, 1, 5])
@pytest.mark.parametrize("checksum", [True, False])
def test_the_archive_is_compress_seekables(pkg, ctx, data, monkeypatch, kind, level, checksum):
    per_group = (2 if level else 0) + (1 if checksum else 0) + 2   # k_cmatch, k_cenc, k_cxxh64, k_cscan, k_cassemble
    for fs in FRAME_SIZES:
        for n in lengths(fs):
            plain = data[kind][:n]
            want = pkg.compress_seekable(ctx, plain, frame_size=fs, level=level, checksum=checksum)
            for chunk in CHUNKS:
                set_chunk(monkeypatch, chunk)
                before = ctx.kernel_launches()
                got, r = stream(pkg, ctx, plain, fs, level, checksum, seed=n + chunk)
                assert got == want, (fs, n, chunk)
                assert r["groups"] == groups_of(n, fs, chunk), (fs, n, chunk)
                assert ctx.kernel_launches() - before == r["groups"] * per_group + 1   # and one k_cseek


def test_a_frame_larger_than_the_default_chunk(pkg, ctx, data, monkeypatch):
    fs = DEFAULT + 5
    plain = (data["c2b"] * (fs // len(data["c2b"]) + 2))[:fs + 1000]
    monkeypatch.delenv(ENV, raising=False)
    got, r = stream(pkg, ctx, plain, fs, seed=7)
    assert r["groups"] == 2 and r["frames"] == 2
    assert got == pkg.compress_seekable(ctx, plain, frame_size=fs)


@pytest.fixture(scope="module")
def dicts(pkg, ctx, data):
    content = datagen.gen_text(65536, 0x5E53).tobytes()
    samples = [data["c2b"][i:i + 20000] for i in range(0, 400000, 20000)]
    return {"raw": pkg.Dictionary.raw_content(ctx, 1, content), "formatted": pkg.Dictionary.decode_dict(ctx, pkg.finalize_dict(ctx, content, samples)),
            "content": content}


@pytest.mark.parametrize("which", ["raw", "formatted", "formatted_tables"])
@pytest.mark.parametrize("level", [1, 5])
def test_with_dictionaries(pkg, ctx, data, dicts, monkeypatch, which, level):
    D = dicts["raw" if which == "raw" else "formatted"]
    tables = which == "formatted_tables"
    plain = data["c2b"][:700_001]
    for fs in (4103, 100_000):
        want = pkg.compress_seekable(ctx, plain, frame_size=fs, level=level, dict=D, dict_tables=tables)
        for chunk in (131072, DEFAULT):
            set_chunk(monkeypatch, chunk)
            got, _ = stream(pkg, ctx, plain, fs, level, dict=D, dict_tables=tables, seed=fs + chunk)
            assert got == want, (fs, chunk)


@pytest.mark.parametrize("level", [0, 1, 5])
def test_round_trip(pkg, ctx, oracle, data, monkeypatch, level):
    plain = data["silesia"][:1_000_003]
    set_chunk(monkeypatch, 1 << 20)
    arch, _ = stream(pkg, ctx, plain, 131072, level, seed=3)
    out = np.zeros(len(plain) + 64, dtype=np.uint8)
    s, _ = pkg.decode_all(ctx, arch, out)
    assert s["status"] == 0 and s["written"] == len(plain) and out[:len(plain)].tobytes() == plain
    assert datagen.decompress(arch, len(plain) + 64) == plain
    assert bytes(oracle.FrameDecoder().decode_all(arch, len(plain) + 64)) == plain


def test_argument_checks(pkg, ctx, data):
    plain = data["c2b"][:10000]
    before = ctx.kernel_launches()
    for fs, level, code in ((0, 1, 220), ((1 << 30) + 1, 1, 220), (4096, 6, 220), (4096, 3, 200), (4096, 2, 200)):
        src, drain = Source(plain), Drain()
        with pytest.raises(pkg.B200ZError) as e:
            pkg.compress_seekable_stream(ctx, src, drain, fs, level)
        assert e.value.code == code and src.calls == 0 and drain.calls == 0, (fs, level)
    assert ctx.kernel_launches() == before


@pytest.mark.parametrize("side", ["source", "drain", "drain_full"])
def test_failing_callbacks(pkg, ctx, data, monkeypatch, side):
    plain = data["c2b"][:1_200_000]
    set_chunk(monkeypatch, 131072)
    fresh = pkg.Context(0)
    try:
        want, _ = stream(pkg, fresh, plain, 4103, seed=11)
    finally:
        fresh.close()
    src = Source(plain, None, fail_at=4 if side == "source" else None)
    drain = Drain(fail_at=None if side == "source" else 4, full=side == "drain_full")
    with pytest.raises(pkg.B200ZError) as e:
        pkg.compress_seekable_stream(ctx, src, drain, 4103)
    assert e.value.code == pkg.binding.ERR_SEEKABLE_IO
    assert ("read_cb" if side == "source" else "write_cb") in str(e.value) and "archive offset" in str(e.value)
    if side != "drain_full":
        assert isinstance(e.value.__cause__, IOError)
    assert want.startswith(bytes(drain.out))                                      # what was written stays written, and is right
    got, _ = stream(pkg, ctx, plain, 4103, seed=11)
    assert got == want


class Repeat:
    """`plain` `times` times over, without holding more than one copy"""

    def __init__(self, plain, times):
        self.m, self.left, self.pos = memoryview(plain), len(plain) * times, 0

    def read(self, n):
        n = min(n, self.left, len(self.m) - self.pos)
        out = bytes(self.m[self.pos:self.pos + n])
        self.pos = (self.pos + n) % len(self.m)
        self.left -= n
        return out


class Count:
    def __init__(self):
        self.n = 0

    def write(self, b):
        self.n += len(b)
        return len(b)


def test_bounded_memory(pkg, monkeypatch):
    """The library's own count of what its allocations hold (b200z_debug_held_bytes), not a card-wide reading, which other work on a
    shared device moves.  The garbage collector is off between the readings, so that no context or archive an earlier test left in a
    reference cycle is freed in the middle and counted as a change."""
    monkeypatch.delenv(ENV, raising=False)
    ctx = pkg.Context(0)
    plain = datagen.gen_text(64 << 20, 5).tobytes()
    gc.collect()
    gc.disable()
    try:
        dev0, pin0 = pkg.binding.held_bytes()
        r1 = pkg.compress_seekable_stream(ctx, Repeat(plain, 1), Count(), 131072)
        dev1, pin1 = pkg.binding.held_bytes()
        r2 = pkg.compress_seekable_stream(ctx, Repeat(plain, 16), Count(), 131072)
        dev2, pin2 = pkg.binding.held_bytes()
    finally:
        gc.enable()
    assert r1["read"] == len(plain) and r2["read"] == 16 * len(plain) and r2["groups"] == 16
    # what grows with the source is the table: its entries in an array doubled when full (at most 2 * 12 bytes per frame), and the
    # table frame k_cseek writes into the compressor's output staging, which grows by half when it grows (17 + 12 per frame, + 16)
    table = 12 * int(r2["frames"])
    assert 0 <= dev2 - dev1 <= 2 * table + 1.5 * (table + 33), (dev0, dev1, dev2)
    assert pin2 == pin1, (pin1, pin2)
    print(f"compress_seekable_stream holds {dev1 - dev0} bytes of device and {pin1 - pin0} of pinned memory at 64 MiB groups; "
          f"a 1 GiB source adds {dev2 - dev1} device bytes")
    ctx.close()


# ---- reading through a positional-read callback

class Recorder(io.RawIOBase):
    """A file object without a descriptor (so from_source uses seek + read) that records every (offset, length) read and can be made
    to come up short (every read returns nothing) or to raise."""

    def __init__(self, data):
        self.b, self.pos, self.calls, self.short, self.fail = data, 0, [], False, False

    def readable(self):
        return True

    def seekable(self):
        return True

    def seek(self, off, whence=io.SEEK_SET):
        self.pos = off if whence == io.SEEK_SET else len(self.b) + off if whence == io.SEEK_END else self.pos + off
        return self.pos

    def read(self, n=-1):
        self.calls.append((self.pos, n))
        if self.fail:
            raise IOError("archive read failed")
        out = b"" if self.short else self.b[self.pos:self.pos + n]
        self.pos += len(out)
        return out


class Sparse(Recorder):
    """A file of `size` zero bytes that ends with `tail`, never held: reads are made up on demand."""

    def __init__(self, size, tail):
        super().__init__(b"")
        self.size, self.tail = size, tail

    def read(self, n=-1):
        self.calls.append((self.pos, n))
        t0 = self.size - len(self.tail)
        out = bytes(max(0, min(n, t0 - self.pos))) + self.tail[max(0, self.pos - t0):max(0, self.pos + n - t0)]
        self.pos += len(out)
        return out


@pytest.fixture(scope="module")
def archives(pkg, ctx, data):
    from test_seekable_model import libzstd_archive
    return [(pkg.compress_seekable(ctx, data["c2b"], frame_size=131072), data["c2b"]),
            (pkg.compress_seekable(ctx, data["silesia"], frame_size=50_000, level=5, checksum=False), data["silesia"]),
            libzstd_archive(0x5E3, True)]


def range_sets(arch, plain, rng):
    entries, _ = seekable.parse(arch)
    sets = list(seekable.crafted_ranges(entries).values())
    sets.append(seekable.random_ranges(len(plain), 2000, rng, 1, 65536)[0])
    return sets


def read_both(pkg, ctx, a, b, rs, dev):
    end = max(oo + ln for _, ln, oo in rs) + 8
    outs = []
    res = []
    for x in (a, b):
        out = torch.full((end,), 0xEE, dtype=torch.uint8, device="cuda") if dev else np.full(end, 0xEE, dtype=np.uint8)
        before = ctx.kernel_launches()
        res.append((x.read_ranges(rs, out), ctx.kernel_launches() - before))
        outs.append(out.cpu().numpy().tobytes() if dev else out.tobytes())
    return outs, res


def test_from_source_reads_as_the_host_archive(pkg, ctx, archives, tmp_path):
    rng = np.random.default_rng(0x5E54)
    for k, (arch, plain) in enumerate(archives):
        path = tmp_path / f"a{k}.zst"
        path.write_bytes(arch)
        for flags in (0, pkg.binding.FLAG_CHECKSUM):
            ctx.set_flags(flags)
            try:
                with pkg.SeekableArchive.from_source(ctx, str(path)) as f, pkg.SeekableArchive(ctx, arch) as m:
                    assert f.num_frames == m.num_frames and f.content_size == m.content_size == len(plain)
                    assert np.array_equal(f.frames, m.frames)
                    for rs in range_sets(arch, plain, rng):
                        for dev in (False, True):
                            (got, want), ((rf, lf), (rm, lm)) = read_both(pkg, ctx, f, m, rs, dev)
                            assert got == want and np.array_equal(rf, rm) and lf == lm, (k, flags, dev)
                            assert (rf["status"] == 0).all()
                            for off, ln, oo in rs[:64]:
                                assert got[oo:oo + ln] == plain[off:off + ln]
            finally:
                ctx.set_flags(0)
    arch, plain = archives[0]
    with pkg.SeekableArchive.from_source(ctx, io.BytesIO(arch)) as f:   # no descriptor: seek + read
        assert f.read(123_457, 300_000) == plain[123_457:423_457]
    with open(tmp_path / "a0.zst", "rb") as fh, pkg.SeekableArchive.from_source(ctx, fh) as f:
        assert f.read(5, 100) == plain[5:105]


def test_what_the_callback_is_asked_for(pkg, ctx, archives):
    rng = np.random.default_rng(0x5E55)
    for arch, plain in archives:
        entries, ck = seekable.parse(arch)
        tb = 17 + len(entries) * (12 if ck else 8)
        rec = Recorder(arch)
        with pkg.SeekableArchive.from_source(ctx, rec, len(arch)) as f:
            assert rec.calls == [(len(arch) - 9, 9), (len(arch) - tb, 8), (len(arch) - tb, tb)]   # footer, table header, table
            for rs in range_sets(arch, plain, rng):
                rec.calls.clear()
                out = np.zeros(max(oo + ln for _, ln, oo in rs) + 8, dtype=np.uint8)
                assert (f.read_ranges(rs, out)["status"] == 0).all()
                frames, _, _ = pkg.seekable_plan(arch, rs)
                runs = []
                for fi in sorted(int(x) for x in frames["frame"]):
                    off, size = entries[fi][0], entries[fi][1]
                    if runs and runs[-1][0] + runs[-1][1] == off:
                        runs[-1][1] += size
                    else:
                        runs.append([off, size])
                assert rec.calls == [tuple(r) for r in runs]


def test_bad_sources(pkg, ctx, archives):
    arch, plain = archives[0]
    entries, _ = seekable.parse(arch)
    at = len(arch) - (17 + 12 * len(entries))

    def corrupt(off, val):
        b = bytearray(arch)
        b[off] = val
        return bytes(b)
    bad = [arch[:16], corrupt(len(arch) - 1, 0), corrupt(len(arch) - 5, 0x84), corrupt(at, 0), corrupt(at + 4, 0),
           corrupt(at + 8, arch[at + 8] ^ 1), arch[:-1]]
    for b in bad:
        with pytest.raises(pkg.B200ZError) as mem:
            pkg.SeekableArchive(ctx, b)
        with pytest.raises(pkg.B200ZError) as src:
            pkg.SeekableArchive.from_source(ctx, io.BytesIO(b))
        assert mem.value.code == src.value.code == pkg.binding.ERR_SEEKABLE_TABLE and str(mem.value) == str(src.value)
    rec = Recorder(arch)
    rec.short = True
    with pytest.raises(pkg.B200ZError) as e:
        pkg.SeekableArchive.from_source(ctx, rec, len(arch))
    assert e.value.code == pkg.binding.ERR_SEEKABLE_IO
    rec = Recorder(arch)
    with pkg.SeekableArchive.from_source(ctx, rec, len(arch)) as f:
        for how in ("short", "fail"):
            setattr(rec, how, True)
            before = ctx.kernel_launches()
            with pytest.raises(pkg.B200ZError) as e:
                f.read(200_000, 5000)
            assert e.value.code == pkg.binding.ERR_SEEKABLE_IO and "archive offset" in str(e.value)
            assert ctx.kernel_launches() == before
            if how == "fail":
                assert isinstance(e.value.__cause__, IOError)
            setattr(rec, how, False)
            assert f.read(200_000, 5000) == plain[200_000:205_000]
    # a 200 GB archive whose footer claims 2^32 - 1 frames with checksums: the table frame's header is read and refused before
    # anything of the claimed table's size (about 51 GB) is allocated or read
    huge = 200 << 30
    sparse = Sparse(huge, struct.pack("<IBI", 0xFFFFFFFF, 0x80, seekable.FOOTER_MAGIC))
    with pytest.raises(pkg.B200ZError) as e:
        pkg.SeekableArchive.from_source(ctx, sparse, huge)
    assert e.value.code == pkg.binding.ERR_SEEKABLE_TABLE
    tb = 17 + 12 * 0xFFFFFFFF
    assert sparse.calls == [(huge - 9, 9), (huge - tb, 8)]
    with pytest.raises(pkg.B200ZError) as e:   # a length past the file's end: the footer read comes up short
        pkg.SeekableArchive.from_source(ctx, io.BytesIO(arch), len(arch) + 10)
    assert e.value.code == pkg.binding.ERR_SEEKABLE_IO
