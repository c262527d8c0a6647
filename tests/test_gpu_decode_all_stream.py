"""decode_all from a reader to a writer (b200z_decode_all_stream, tier 1d), checked against the oracle's FrameDecoder.decode_all for the
output and against b200z_decode_all_batch for the outcome, at chunk sizes that put frames across many submissions."""
import random

import numpy as np
import pytest

from conftest import read_golden
from test_decode_all_chain import concat_with_skippables, corpus_frames, skippable

pytestmark = pytest.mark.gpu

SUMMARY = ("written", "frames", "skippable_frames", "error_offset", "status", "stage", "error_frame")
DEFAULT = 64 << 20


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


class Source:
    """A reader that hands out the bytes whole, one byte per call, or in seeded random lengths; optionally raising at call n."""

    def __init__(self, data, reads="whole", fail_at=None):
        self.b, self.pos, self.calls, self.fail_at = data, 0, 0, fail_at
        self.rng = random.Random(reads) if isinstance(reads, int) else None
        self.reads = reads

    def read(self, n):
        self.calls += 1
        if self.fail_at is not None and self.calls >= self.fail_at:
            raise IOError("source failed")
        if self.reads == "byte":
            n = min(n, 1)
        elif self.rng is not None:
            n = min(n, self.rng.choice([1, 3, 17, 4096, 65536, 1 << 20]))
        out = self.b[self.pos:self.pos + n]
        self.pos += len(out)
        return out


class Drain:
    """A writer that returns 0 at call `full_at` (the drain is full)."""

    def __init__(self, full_at=None):
        self.out, self.calls, self.full_at = bytearray(), 0, full_at

    def write(self, b):
        self.calls += 1
        if self.full_at is not None and self.calls >= self.full_at:
            return 0
        self.out += b
        return len(b)


def stream(pkg, ctx, monkeypatch, data, chunk=DEFAULT, reads="whole", **kw):
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(chunk))
    d = Drain()
    r = pkg.decode_all_stream(ctx, Source(data, reads), d, **kw)
    assert r["delivered"] == len(d.out)
    return r, bytes(d.out)


def batch(pkg, ctx, data, cap, **kw):
    return pkg.decode_all_batch(ctx, data, np.zeros(max(cap, 1) + 16, dtype=np.uint8)[:max(cap, 1)], **kw)


def oracle_all(oracle, data, cap, dict_raw=None):
    d = oracle.FrameDecoder()
    if dict_raw is not None:
        d.add_dict(dict_raw)
    try:
        return d.decode_all(data, cap)
    except oracle.OracleError:
        return None


def check(pkg, ctx, oracle, monkeypatch, data, cap, chunk=DEFAULT, reads="whole", dict_raw=None, **kw):
    r, out = stream(pkg, ctx, monkeypatch, data, chunk, reads, **kw)
    want = batch(pkg, ctx, data, cap, **kw)
    assert {k: r[k] for k in SUMMARY} == want, (chunk, reads)
    exp = oracle_all(oracle, data, cap, dict_raw)
    if exp is not None:
        assert r["status"] == 0 and out == exp, (chunk, reads, len(out), len(exp))
    assert r["delivered"] >= r["written"]
    return r, out


@pytest.mark.parametrize("chunk", [4096, 131072, 1 << 20, DEFAULT])
def test_corpus_with_skippables(pkg, ctx, oracle, manifest, exec_mode, monkeypatch, chunk):
    frames = corpus_frames(manifest)
    buf, _ = concat_with_skippables(frames)
    total = 64 << 20
    for reads in ("whole", 7):
        r, _ = check(pkg, ctx, oracle, monkeypatch, buf, total, chunk, reads)
        assert r["frames"] == len(frames) and r["status"] == 0
    if chunk == 131072:
        small, _ = concat_with_skippables(frames[:6])
        check(pkg, ctx, oracle, monkeypatch, small, total, chunk, "byte")


def compressor_frame(pkg, ctx, plain):
    out = bytearray()
    pkg.compress(ctx, plain, out)
    return bytes(out)


@pytest.mark.parametrize("chunk", [131072, DEFAULT])
def test_stream_compressor_frames_and_checksums(pkg, ctx, exec_mode, monkeypatch, chunk):
    import datagen as G
    plain = G.gen_text(5 << 20, 71).tobytes()
    frame = compressor_frame(pkg, ctx, plain)
    flags = ctx.L.b200z_ctx_flags(ctx.h)
    try:
        for flag in (0, 1):
            ctx.set_flags(flags | flag)
            n0 = ctx.kernel_launches()
            r, out = stream(pkg, ctx, monkeypatch, frame, chunk)
            launched = ctx.kernel_launches() - n0
            assert r["status"] == 0 and out == plain and r["frames"] == 1
            if chunk == 131072:
                assert r["submissions"] >= 10   # a few blocks per submission: the frame is carried across all of them
            if exec_mode == "warp":   # a decode_all pass is 6 kernels there; k_carry per continuing frame; the hash per submission
                assert launched == r["submissions"] * (6 + flag) + (r["submissions"] - 1), (launched, r)
            if flag:
                assert r["checksum_frames"] == 1 and r["checksum_mismatches"] == 0 and r["first_mismatch_frame"] == -1
            bad = frame[:-4] + bytes(b ^ 0xFF for b in frame[-4:])
            r2, out2 = stream(pkg, ctx, monkeypatch, bad, chunk)
            assert r2["status"] == 0 and out2 == plain
            if flag:
                assert r2["checksum_mismatches"] == 1 and r2["first_mismatch_frame"] == 0
    finally:
        ctx.set_flags(flags)


def test_checksums_of_many_frames(pkg, ctx, oracle, manifest, exec_mode, monkeypatch):
    import datagen as G
    frames = [G.compress(G.gen_text(n, 90 + n), checksum=True) for n in (2, 31, 32, 33, 1000, 300000, 1 << 20)]
    buf = b"".join(frames) + skippable(5) + frames[-1]
    flags = ctx.L.b200z_ctx_flags(ctx.h)
    try:
        ctx.set_flags(flags | 1)
        for chunk in (4096, 131072, DEFAULT):
            r, _ = check(pkg, ctx, oracle, monkeypatch, buf, 8 << 20, chunk)
            assert r["checksum_frames"] == len(frames) + 1 and r["checksum_mismatches"] == 0
    finally:
        ctx.set_flags(flags)


@pytest.mark.parametrize("window_log", [20, 21, 22, 23])
def test_windows_longer_than_a_chunk(pkg, ctx, oracle, exec_mode, monkeypatch, window_log):
    import datagen as G
    plain = G.gen_text(6 << 20, window_log).tobytes()
    frame = G.compress(plain, level=3, window_log=window_log)
    for chunk in (131072, 1 << 20):
        r, out = check(pkg, ctx, oracle, monkeypatch, frame, len(plain), chunk)
        assert out == plain
    mix = G.gen_silesia_mix(4 << 20, window_log).tobytes()
    frame = G.compress(mix, level=3, window_log=window_log)
    r, out = check(pkg, ctx, oracle, monkeypatch, frame + frame, 2 * len(mix), 262144)
    assert out == mix + mix


def test_dictionaries(pkg, ctx, oracle, manifest, exec_mode, monkeypatch):
    dic = read_golden("dict_tests", "dictionary")
    names = sorted(manifest["dict"])
    frames = [read_golden("dict_tests", "files", n) for n in names]
    buf = b"".join(frames)
    D = pkg.Dictionary.decode_dict(ctx, dic)
    total = sum(manifest["dict"][n]["size"] for n in names)
    for chunk in (4096, DEFAULT):
        r, _ = check(pkg, ctx, oracle, monkeypatch, buf, total, chunk, dict_raw=dic, dicts=[D])
        assert r["frames"] == len(frames)
    r, _ = stream(pkg, ctx, monkeypatch, buf, DEFAULT)
    assert r["status"] != 0 and pkg.error_names()[r["status"]] == "B200Z_ERR_DICT_NOT_PROVIDED"


def test_forced_raw_content_dictionary(pkg, ctx, exec_mode, monkeypatch):
    import datagen as G
    fs = G.config_c5(nframes=300, cache=False)
    D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict)
    for chunk in (4096, DEFAULT):
        r, out = stream(pkg, ctx, monkeypatch, fs.comp.tobytes(), chunk, forced_dict=D)
        assert r["status"] == 0 and out == fs.plain.tobytes()[:fs.D]


def oracle_delivered(oracle, data, r):
    """What the drain must hold after the error `r` reports: the frames before the failing one, then the failing frame's output of
    every block before its first failing block, as the oracle's FrameDecoder finds it decoding UptoBlocks(1) block after block."""
    if r["status"] == 0 or r["error_frame"] < 0:
        return r["written"]
    d = oracle.FrameDecoder()
    d.trace_enable()
    try:
        rd = d.reset(data[r["error_offset"]:])
        while not d.is_finished():
            d.decode_blocks(rd, oracle.UPTO_BLOCKS, 1)
    except oracle.OracleError:
        pass
    blocks = d.trace()[0]
    return r["written"] + sum(b["out_size"] for b in blocks[:d.blocks_decoded()])


def test_truncations_and_garbage(pkg, ctx, oracle, manifest, exec_mode, monkeypatch):
    frames = corpus_frames(manifest)[:12]
    buf, starts = concat_with_skippables(frames)
    full_out = oracle_all(oracle, buf, 16 << 20)
    # inside each frame too: after its header, between blocks, inside a block and just before its checksum
    inner = {s + int(f * len(frames[i // 2])) for i, s in enumerate(starts) if i % 2 == 0 for f in (0.3, 0.6, 0.9)}
    cuts = sorted(({s + d for s in starts for d in (-3, -1, 1, 5, 40)} | inner | {len(buf) // 3, len(buf) // 2}) & set(range(1, len(buf))))
    for chunk in (4096, DEFAULT):
        for n in cuts:
            r, out = check(pkg, ctx, oracle, monkeypatch, buf[:n], 16 << 20, chunk)
            assert out == full_out[:oracle_delivered(oracle, buf[:n], r)], (n, chunk, r)
        for tail in (b"\x00", b"garbage that is no frame", b"\x28\xb5\x2f\xfd", b"\x50\x2a\x4d\x18\x00\x00"):
            r, out = check(pkg, ctx, oracle, monkeypatch, buf + tail, 16 << 20, chunk)
            assert r["status"] != 0 and out == full_out
            assert len(out) == oracle_delivered(oracle, buf + tail, r)


def test_corrupt_block_in_a_frame_across_submissions(pkg, ctx, oracle, exec_mode, monkeypatch):
    import datagen as G
    plain = G.gen_text(2 << 20, 5).tobytes()
    frame = bytearray(compressor_frame(pkg, ctx, plain))
    # the 9th block of the frame: walk the block headers
    pos, k = 6, 0
    while k < 8:
        h = int.from_bytes(frame[pos:pos + 3], "little")
        pos += 3 + (1 if (h >> 1) & 3 == 1 else h >> 3)
        k += 1
    h = int.from_bytes(frame[pos:pos + 3], "little")
    assert (h >> 1) & 3 == 2, "the 9th block is Compressed"
    frame[pos + 3:pos + 3 + (h >> 3)] = bytes(0xFF for _ in range(h >> 3))
    lead = compressor_frame(pkg, ctx, plain[:1000])
    data = lead + bytes(frame)
    for chunk in (131072, 1 << 20, DEFAULT):
        r, out = stream(pkg, ctx, monkeypatch, data, chunk)
        want = batch(pkg, ctx, data, 4 << 20)
        assert {k: r[k] for k in SUMMARY} == want
        assert r["status"] != 0 and r["error_frame"] == 1 and r["written"] == 1000
        assert out == plain[:1000] + plain[:8 * 131072]   # the failing frame's output before its failing block
        assert len(out) == oracle_delivered(oracle, data, r)


def test_failing_source_and_drain(pkg, ctx, oracle, manifest, exec_mode, monkeypatch):
    buf, _ = concat_with_skippables(corpus_frames(manifest)[:30])
    full = stream(pkg, ctx, monkeypatch, buf, 4096)[1]
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", "4096")
    for n in (1, 2, 5):
        d = Drain(full_at=n)
        r = pkg.decode_all_stream(ctx, Source(buf, 3), d)
        assert pkg.error_names()[r["status"]] == "B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER" and r["stage"] == 9
        assert full.startswith(bytes(d.out)) and r["delivered"] == len(d.out)
        assert stream(pkg, ctx, monkeypatch, buf, 4096)[1] == full   # the context is still right
    for n in (2, 9):
        d = Drain()
        src = Source(buf, 3, fail_at=n)
        r = pkg.decode_all_stream(ctx, src, d)
        consumed = src.pos
        want = batch(pkg, ctx, buf[:consumed], 16 << 20)
        assert {k: r[k] for k in SUMMARY} == want
        assert full.startswith(bytes(d.out))
        assert stream(pkg, ctx, monkeypatch, buf, 4096)[1] == full


def device_bytes_used():
    """(device memory this process uses, exact): NVML's per-process figure when NVML can see this process; otherwise (the
    card's used memory, False), which other processes on a shared card move too."""
    import os
    import torch
    torch.cuda.synchronize()
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        for p in pynvml.nvmlDeviceGetComputeRunningProcesses(h):
            if p.pid == os.getpid() and p.usedGpuMemory is not None:
                return int(p.usedGpuMemory), True
    except Exception:
        pass
    free, total = torch.cuda.mem_get_info()
    return total - free, False


def test_bounded_memory(pkg, monkeypatch):
    import datagen as G
    ctx = pkg.Context(0)
    plain = G.gen_text(64 << 20, 3).tobytes()
    frame = compressor_frame(pkg, ctx, plain)
    used0, _ = device_bytes_used()
    r, out = stream(pkg, ctx, monkeypatch, frame, DEFAULT)
    assert r["status"] == 0 and len(out) == len(plain)
    used1, exact = device_bytes_used()
    r, _ = stream(pkg, ctx, monkeypatch, frame * 16, DEFAULT)
    assert r["status"] == 0 and r["written"] == 16 * len(plain)
    used2, exact2 = device_bytes_used()
    # the context's buffers depend on the chunk and the largest window only; a card-wide reading also moves with other processes
    # (a slot sized by the stream's length would differ by 4 * C = 256 MiB)
    assert abs(used2 - used1) <= (0 if exact and exact2 else 16 << 20), (used1, used2, exact)
    C, W = DEFAULT, 131072
    assert used1 - used0 <= 2 * (12.5 * C + W) + (64 << 20), used1 - used0
    print(f"decode_all_stream holds {used1 - used0} bytes of device memory at {C}-byte chunks (per process: {exact})")
    ctx.close()


def dictionary_cross_cases():
    """tests/dictcraft.py frames of several blocks whose later blocks reach into the dictionary: Raw and RLE blocks (not counted
    by total_output_counter) between Compressed blocks that each copy a match wholly from the dictionary and then straddle its end
    and the frame's first bytes.  At a 4096-byte chunk every block is its own submission, so each reach comes from a frame resumed
    behind its carried tail, with its dictionary and its tables carried."""
    import dictcraft as D
    rng = random.Random(0x5D1C)
    out = []
    for dct, forced in ((D.D_MAIN, None), (D.D_LONG, None), (D.D_R, D.D_R)):
        dl = len(dct.content)
        blocks, p = [], 0
        for k in range(4):
            raw = rng.randbytes(700 + 300 * k)
            blocks += [("raw", raw), ("rle", 0x41 + k, 257)]
            p += len(raw) + 257
            full = min(dl, 40 + 30 * k)
            seqs = [(3, 20, D._new(p + 3 + full)), (2, 30, D._new(p + 3 + 20 + 2 + 10))]
            seqs += D._ordinary(rng, 4, p + 3 + 20 + 2 + 30)
            blocks.append(("cmp", D._lits(rng, seqs, 5), seqs))
            p += sum(q[0] + q[1] for q in seqs) + 5
        out.append(D.Case("stream", f"dict-across-cuts-{dct.name}", blocks, dict=None if forced else dct, forced=forced))
    return out


def test_dictionary_reach_across_submissions(pkg, ctx, oracle, exec_mode, monkeypatch):
    import dictcraft as D
    handles = {d.name: (pkg.Dictionary.decode_dict(ctx, d.raw) if d.formatted else pkg.Dictionary.raw_content(ctx, d.id, d.content))
               for d in (D.D_MAIN, D.D_LONG, D.D_R)}
    named = [handles[D.D_MAIN.name], handles[D.D_LONG.name]]
    for c in dictionary_cross_cases():
        assert c.valid and sum(1 for x in c.full.reaches if x[0] >= 3) >= 6, c   # reaches in the frame's later blocks
        forced = handles[c.forced.name] if c.forced is not None else None
        data = c.frame + skippable(3) + c.frame
        exp = c.expected * 2
        if forced is None:
            assert D.oracle_decoder(oracle).decode_all(data, len(exp)) == exp
        for chunk in (4096, 131072, DEFAULT):
            r, out = stream(pkg, ctx, monkeypatch, data, chunk, dicts=named, forced_dict=forced)
            assert {k: r[k] for k in SUMMARY} == batch(pkg, ctx, data, len(exp), dicts=named, forced_dict=forced), (c, chunk)
            assert r["status"] == 0 and out == exp, (c, chunk)
            if chunk == 4096:
                assert r["submissions"] == 2 * len(c.blocks), (c, r)
