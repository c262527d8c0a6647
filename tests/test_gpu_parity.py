"""GPU parity tests: the CUDA path (through the C ABI) against the oracle and the reference's golden vectors.
Bit-exact everywhere -- the whole path is integer / byte work."""
import hashlib
import os

import numpy as np
import pytest

import intermediates
from conftest import read_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["cta", "warp"])
def exec_mode(request, monkeypatch):
    """Which LZ77 execution kernel takes the frames: k_exec_cta (block assembled in shared memory, falls back to the warp kernel
    per block for what it does not handle) or k_exec (one warp per frame) for everything.  Tests without this fixture run the
    shipped default (auto: by frame size / dictionary)."""
    monkeypatch.setenv("B200Z_EXEC_MODE", request.param)
    return request.param


def _io(pkg, frames, sizes, slack=0):
    io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, (f, n) in enumerate(zip(frames, sizes)):
        io[i] = (so, len(f), oo, n + slack)
        so += len(f); oo += n + slack
    return io, np.frombuffer(b"".join(frames), dtype=np.uint8), oo


def test_corpus_frame_decoder(pkg, ctx, manifest, exec_mode):
    """tests/decode_corpus.rs through the FrameDecoder mirror: reset + decode_blocks(All) + collect."""
    dec = pkg.FrameDecoder(ctx)
    for name, m in manifest["corpus"].items():
        data = read_golden("decodecorpus", name)
        r = dec.reset(data)
        assert dec.decode_blocks(r, pkg.ALL) is True
        out = dec.collect()
        assert len(out) == m["size"], name
        assert hashlib.sha256(out).hexdigest() == m["sha256"], name
        assert dec.bytes_read_from_source() == len(data), name
        assert dec.get_checksum_from_data() == dec.get_calculated_checksum() == m["xxh64_low32"], name
        assert dec.is_finished()


def test_corpus_batch_and_intermediates(pkg, ctx, oracle, manifest, exec_mode):
    """All 101 frames in ONE submission; per-block literals and sequences against the oracle's trace."""
    names = sorted(manifest["corpus"])
    frames = [read_golden("decodecorpus", n) for n in names]
    sizes = [manifest["corpus"][n]["size"] for n in names]
    io, comp, total = _io(pkg, frames, sizes)
    import torch
    d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, comp, io)
    b.run(d_out)
    res = b.finish()
    out = d_out.cpu().numpy()
    blk = 0
    nlit = nseq = 0
    for i, n in enumerate(names):
        assert res[i]["status"] == 0, (n, res[i])
        assert res[i]["out_size"] == sizes[i] and res[i]["bytes_read"] == len(frames[i]), n
        got = out[io[i]["out_off"]:io[i]["out_off"] + sizes[i]].tobytes()
        assert hashlib.sha256(got).hexdigest() == manifest["corpus"][n]["sha256"], n
        assert res[i]["has_checksum"] == 1 and res[i]["checksum_from_data"] == manifest["corpus"][n]["xxh64_low32"]
        d = oracle.FrameDecoder(); d.trace_enable()
        r = d.reset(frames[i]); d.decode_blocks(r); d.collect()
        blocks, lits, seqs = d.trace()
        assert res[i]["blocks_decoded"] == len(blocks)
        blk, nl, ns = intermediates.check_intermediates(b, blk, blocks, lits, seqs, n)
        nlit += nl
        nseq += ns
    assert nlit > 1000 and nseq > 1_000_000   # 2458 compressed blocks / 1,031,936 sequences in the corpus


def test_gpu_checksum_stage(pkg, manifest):
    """B200Z_FLAG_CHECKSUM: XXH64 on the GPU == the stored content checksum for all 101 corpus frames (tests/decode_corpus.rs:61-74),
    incl. empty and tiny frames, and == the host hash for random lengths around the 32-byte stripe boundary."""
    import torch
    c2 = pkg.Context(0)
    c2.set_flags(pkg.binding.FLAG_CHECKSUM)
    names = sorted(manifest["corpus"])
    frames = [read_golden("decodecorpus", n) for n in names]
    sizes = [manifest["corpus"][n]["size"] for n in names]
    io, comp, total = _io(pkg, frames, sizes)
    d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(c2, comp, io)
    b.run(d_out)
    res = b.finish()
    for i, n in enumerate(names):
        assert res[i]["status"] == 0 and res[i]["has_calculated_checksum"] == 1, n
        assert res[i]["calculated_checksum"] == res[i]["checksum_from_data"] == manifest["corpus"][n]["xxh64_low32"], n
    import datagen as G
    rng = np.random.Generator(np.random.PCG64(9))
    pieces = [rng.integers(0, 256, int(n), dtype=np.uint8) for n in list(range(0, 70)) + [255, 256, 257, 4095, 4096, 4097, 65537]]
    frames = [G.compress(p_, level=1) for p_ in pieces]
    io, comp, total = _io(pkg, frames, [len(p_) for p_ in pieces])
    out = np.zeros(total + 64, dtype=np.uint8)
    res = pkg.decode_frames(c2, comp, io, out)
    for i, p_ in enumerate(pieces):
        assert res[i]["status"] == 0 and res[i]["calculated_checksum"] == (pkg.xxh64(p_.tobytes()) & 0xFFFFFFFF) == res[i]["checksum_from_data"], len(p_)
    c2.close()


def test_kernel_launch_counts(pkg, monkeypatch):
    """ctx.kernel_launches() counts the kernels each path really launched, on single-block frames.  The warp kernel takes every
    frame: k_exec_cta would add its own launches."""
    import torch
    import datagen as G
    monkeypatch.setenv("B200Z_EXEC_MODE", "warp")
    plains = [G.gen_text(20000, 70 + i).tobytes() for i in range(8)]
    frames = [G.compress(p_) for p_ in plains]
    c2 = pkg.Context(0)
    dec = pkg.FrameDecoder(c2)
    r = dec.reset(frames[0])
    n0 = c2.kernel_launches()
    assert dec.decode_blocks(r, pkg.ALL) is True
    assert c2.kernel_launches() - n0 == 4   # k_setup, k_huf, k_fse; then k_exec once the output has grown
    assert dec.collect() == plains[0]
    del dec
    io, comp, total = _io(pkg, frames, [len(p_) for p_ in plains])
    d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(c2, comp, io)
    assert b.info()["compressed_blocks"] == len(frames) and b.info()["launches_per_run"] == 0
    n0 = c2.kernel_launches()
    b.run_profile(d_out)
    assert c2.kernel_launches() - n0 == 4   # k_setup, k_huf, k_fse, k_exec, one after the other
    c2.set_flags(pkg.binding.FLAG_CHECKSUM)
    n0 = c2.kernel_launches()
    b.run(d_out)
    assert c2.kernel_launches() - n0 == b.info()["launches_per_run"] == 6   # two k_setup halves, k_huf, k_fse, k_exec, k_xxh64
    res = b.finish()
    assert (res["status"] == 0).all() and (res["has_calculated_checksum"] == 1).all()
    b.close()
    c2.close()


def test_dict_corpus(pkg, ctx, manifest):
    """tests/dict_test.rs:77-262 via the mirror, then all 207 frames in one batch."""
    dic = read_golden("dict_tests", "dictionary")
    dec = pkg.FrameDecoder(ctx)
    dec.add_dict(dic)
    names = sorted(manifest["dict"])
    for name in names:   # all 207 (tests/dict_test.rs:77-262)
        data = read_golden("dict_tests", "files", name)
        r = dec.reset(data)
        dec.decode_blocks(r, pkg.ALL)
        out = dec.collect()
        m = manifest["dict"][name]
        assert len(out) == m["size"] and hashlib.sha256(out).hexdigest() == m["sha256"], name
        assert dec.bytes_read_from_source() == len(data)
    D = pkg.Dictionary.decode_dict(ctx, dic)
    assert D.id == 618557512
    frames = [read_golden("dict_tests", "files", n) for n in names]
    sizes = [manifest["dict"][n]["size"] for n in names]
    io, comp, total = _io(pkg, frames, sizes)
    out = np.zeros(total + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, comp, io, out, dicts=[D])
    for i, n in enumerate(names):
        assert res[i]["status"] == 0 and res[i]["has_dict_id"] == 1 and res[i]["dict_id"] == 618557512, n
        got = out[io[i]["out_off"]:io[i]["out_off"] + res[i]["out_size"]].tobytes()
        assert hashlib.sha256(got).hexdigest() == manifest["dict"][n]["sha256"], n
    # without the dictionary: DictNotProvided, like FrameDecoder::reset (frame_decoder.rs:212-216)
    res = pkg.decode_frames(ctx, comp, io, out)
    assert all(pkg.error_names()[int(s)] == "B200Z_ERR_DICT_NOT_PROVIDED" for s in res["status"])


def test_dictionary_kat(pkg, ctx):
    from test_oracle_kat import DICT_KAT_CONTENT, dict_kat_bytes
    raw = dict_kat_bytes()
    D = pkg.Dictionary.decode_dict(ctx, raw)
    assert D.id == 0x47232101 and D.offset_hist == [3, 10, 0xABCDEF] and D.content_size == len(DICT_KAT_CONTENT)
    with pytest.raises(pkg.B200ZError) as e:
        pkg.Dictionary.decode_dict(ctx, b"\x01\x01\x01\x01" + raw[4:])
    assert pkg.error_names()[e.value.code] == "B200Z_ERR_DICT_BAD_MAGIC_NUM"
    for cut in range(0, len(raw) - len(DICT_KAT_CONTENT), 3):
        with pytest.raises(pkg.B200ZError):
            pkg.Dictionary.decode_dict(ctx, raw[:cut])


def test_fuzz_artifacts_status_parity(pkg, ctx, oracle, manifest, exec_mode):
    """tests/fuzz_regressions.rs: must not crash; and the GPU path must report the SAME outcome as the oracle
    (same error leaf + stage, or the same bytes)."""
    zo, bz = oracle.error_names(), pkg.error_names()
    for sub, files in manifest["fuzz"].items():
        for f in files:
            data = read_golden("fuzz", sub, f)
            try:
                exp, _ = oracle.decode_frame(data)
                exp_err = None
            except oracle.OracleError as e:
                exp, exp_err = None, (zo[e.code].replace("ZO_", ""), e.stage)
            io = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE)
            io[0] = (0, len(data), 0, 1 << 20)
            out = np.zeros((1 << 20) + 16, dtype=np.uint8)
            res = pkg.decode_frames(ctx, np.frombuffer(data, dtype=np.uint8) if data else np.zeros(0, np.uint8), io, out)
            if exp_err is None:
                assert res[0]["status"] == 0, (sub, f, res[0])
                assert out[:res[0]["out_size"]].tobytes() == exp, (sub, f)
            else:
                got = (bz[int(res[0]["status"])].replace("B200Z_", ""), int(res[0]["stage"]))
                assert got == exp_err, (sub, f, got, exp_err)
            dec = pkg.FrameDecoder(ctx)
            try:
                r = dec.reset(data); dec.decode_blocks(r, pkg.ALL); got2 = dec.collect()
                assert exp_err is None and got2 == exp, (sub, f)
            except pkg.B200ZError as e:
                assert exp_err is not None and bz[e.code].replace("B200Z_", "") == exp_err[0], (sub, f, e, exp_err)


def test_fuzz_artifacts_without_dict_id(pkg, ctx, oracle, manifest, exec_mode):
    """Most artifacts stop at DictNotProvided; clear the dict-id flag so the block path itself sees hostile input."""
    zo, bz = oracle.error_names(), pkg.error_names()
    n = 0
    for f in manifest["fuzz"]["decode"]:
        data = bytearray(read_golden("fuzz", "decode", f))
        if len(data) < 6 or data[:4] != bytes([0x28, 0xB5, 0x2F, 0xFD]) or (data[4] & 3) == 0:
            continue
        did = [0, 1, 2, 4][data[4] & 3]
        single = (data[4] >> 5) & 1
        pos = 5 + (0 if single else 1)
        data = bytes(data[:4]) + bytes([data[4] & ~3]) + bytes(data[5:pos]) + bytes(data[pos + did:])
        io = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE)
        io[0] = (0, len(data), 0, 4 << 20)
        out = np.zeros((4 << 20) + 16, dtype=np.uint8)
        # once with the reference's default window limit (WindowSizeTooBig must come out the same), once with the limit lifted on
        # both sides so that the block path itself sees the hostile bytes
        for mw in (0, 1 << 40):
            d = oracle.FrameDecoder()
            if mw:
                d.set_max_window_size(mw)
            try:
                r = d.reset(data); d.decode_blocks(r, oracle.ALL); exp = d.collect(); exp_err = None
            except oracle.OracleError as e:
                exp, exp_err = None, (zo[e.code].replace("ZO_", ""), e.stage)
            res = pkg.decode_frames(ctx, np.frombuffer(data, dtype=np.uint8), io, out, max_window_size=mw)
            if exp_err is None:
                if len(exp) <= 4 << 20:
                    assert res[0]["status"] == 0 and out[:res[0]["out_size"]].tobytes() == exp, (f, mw)
            else:
                got = (bz[int(res[0]["status"])].replace("B200Z_", ""), int(res[0]["stage"]))
                assert got == exp_err, (f, mw, got, exp_err)
        n += 1
    assert n >= 25


def test_window_fixtures(pkg, ctx, manifest, exec_mode):
    """tests/mod.rs:576-741."""
    fox = b"The quick brown fox jumps over the lazy dog.\n" * 4096
    sphinx = b"Sphinx of black quartz, judge my vow.\n" * 4096
    big, small = read_golden("test_fixtures", "window_256mib.zst"), read_golden("test_fixtures", "window_8mib.zst")
    names = pkg.error_names()
    d = pkg.FrameDecoder(ctx); d.set_max_window_size(300 << 20)
    assert d.max_window_size() == 300 << 20
    assert d.decode_all(big, len(fox)) == fox
    d = pkg.FrameDecoder(ctx)
    assert d.max_window_size() == 128 << 20
    with pytest.raises(pkg.B200ZError) as e:
        d.decode_all(big, len(fox))
    assert names[e.value.code] == "B200Z_ERR_WINDOW_SIZE_TOO_BIG"
    d = pkg.FrameDecoder(ctx); d.set_max_window_size(300 << 20)
    assert d.decode_all(big + big, 2 * len(fox)) == fox + fox
    d = pkg.FrameDecoder(ctx)
    with pytest.raises(pkg.B200ZError) as e:
        d.decode_all(small + big, len(fox) + len(sphinx))
    assert names[e.value.code] == "B200Z_ERR_WINDOW_SIZE_TOO_BIG"
    with pytest.raises(pkg.B200ZError) as e:
        pkg.StreamingDecoder(ctx, big)
    assert names[e.value.code] == "B200Z_ERR_WINDOW_SIZE_TOO_BIG"
    s = pkg.StreamingDecoder(ctx, big, max_window_size=300 << 20)
    assert s.read_to_end() == fox
    d = pkg.FrameDecoder(ctx); d.set_max_window_size(2 ** 64 - 1)
    assert d.max_window_size() == (1 << 41) + 7 * (1 << 38)
    assert pkg.FrameDecoder(ctx).decode_all(read_golden("test_fixtures", "window_128mib.zst"), len(fox)) == fox


def test_api_decode_from_to(pkg, ctx, manifest):
    """tests/mod.rs:129-230."""
    content = read_golden("decodecorpus", "z000088.zst")
    d = pkg.FrameDecoder(ctx)
    read1, out1 = d.decode_from_to(content[:50 * 1024], 1 << 20)
    read2, out2 = d.decode_from_to(content[read1:len(content) - 4], 1 << 20)
    assert read1 + read2 == len(content) - 4
    read3, out3 = d.decode_from_to(content[read1 + read2:], 1 << 20)
    assert read3 == 4 and out3 == b""
    res = out1 + out2
    m = manifest["corpus"]["z000088.zst"]
    assert len(res) == m["size"] and hashlib.sha256(res).hexdigest() == m["sha256"]
    assert d.get_checksum_from_data() == d.get_calculated_checksum() == m["xxh64_low32"]


def test_api_streaming_and_reuse(pkg, ctx, manifest):
    """tests/mod.rs:294-380."""
    s = pkg.StreamingDecoder(ctx, read_golden("decodecorpus", "z000088.zst"))
    out = s.read_to_end()
    assert hashlib.sha256(out).hexdigest() == manifest["corpus"]["z000088.zst"]["sha256"]
    s2 = pkg.StreamingDecoder(ctx, read_golden("decodecorpus", "z000068.zst"), decoder=s.into_frame_decoder())
    assert hashlib.sha256(s2.read_to_end()).hexdigest() == manifest["corpus"]["z000068.zst"]["sha256"]


def test_api_streaming_matches_oracle_read_pattern(pkg, ctx, oracle):
    """Same sequence of read() sizes through both StreamingDecoders -> same chunks (window retention, UptoBytes loop)."""
    data = read_golden("decodecorpus", "z000033.zst")
    a, b = pkg.StreamingDecoder(ctx, data), oracle.StreamingDecoder(data)
    rng = np.random.Generator(np.random.PCG64(3))
    while True:
        n = int(rng.integers(1, 200_000))
        x, y = a.read(n), b.read(n)
        assert x == y
        if not y:
            break


def test_api_incremental_read(pkg, ctx):
    """tests/mod.rs:382-404."""
    data = read_golden("decodecorpus", "abc.txt.zst")
    d = pkg.FrameDecoder(ctx)
    r = d.reset(data)
    _, out = d.decode_from_to(r.src.read(), 3)
    assert out == b"abc" and d.is_finished()

    class W:
        def __init__(self): self.buf = bytearray(); self.cap = 3
        def write(self, b):
            k = min(len(b), self.cap - len(self.buf)); self.buf += b[:k]; return k
    w = W()
    assert d.collect_to_writer(w) == 3 and bytes(w.buf) == b"def"


def test_api_decode_all(pkg, ctx, manifest, exec_mode):
    """tests/mod.rs:490-574."""
    def skip(n):
        return (0x184D2A50).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes(n)
    a, b = read_golden("decodecorpus", "z000089.zst"), read_golden("decodecorpus", "z000090.zst")
    inp = skip(300) + a + skip(400) + b + skip(500)
    total = manifest["corpus"]["z000089.zst"]["size"] + manifest["corpus"]["z000090.zst"]["size"]
    names = pkg.error_names()
    d = pkg.FrameDecoder(ctx)
    out = d.decode_all(inp, total)
    assert len(out) == total
    assert hashlib.sha256(out[:manifest["corpus"]["z000089.zst"]["size"]]).hexdigest() == manifest["corpus"]["z000089.zst"]["sha256"]
    with pytest.raises(pkg.B200ZError) as e:
        d.decode_all(inp, total - 1)
    assert names[e.value.code] == "B200Z_ERR_TARGET_TOO_SMALL"
    assert d.decode_all(inp, total + 1) == out
    with pytest.raises(pkg.B200ZError) as e:
        d.decode_all(inp[:-600], total)
    assert e.value.stage == 3      # FrameDecoderError::FailedToReadBlockBody(_)
    with pytest.raises(pkg.B200ZError) as e:
        d.decode_all(inp[:-1], total)
    assert names[e.value.code] == "B200Z_ERR_FAILED_TO_SKIP_FRAME"


def test_strategies_match_oracle(pkg, ctx, oracle, exec_mode):
    """decode_blocks(UptoBlocks / UptoBytes) stop at the same block boundaries and expose the same counters."""
    data = read_golden("decodecorpus", "z000033.zst")
    for strat, n in [(pkg.UPTO_BLOCKS, 7), (pkg.UPTO_BYTES, 5000), (pkg.UPTO_BLOCKS, 0), (pkg.UPTO_BYTES, 300000)]:
        a, b = pkg.FrameDecoder(ctx), oracle.FrameDecoder()
        ra, rb = a.reset(data), b.reset(data)
        for _ in range(2000):
            fa, fb = a.decode_blocks(ra, strat, n), b.decode_blocks(rb, strat, n)
            assert fa == fb
            assert a.blocks_decoded() == b.blocks_decoded() and a.bytes_read_from_source() == b.bytes_read_from_source()
            assert a.can_collect() == b.can_collect()
            k = a.can_collect() // 2
            assert a.read(k) == b.read(k)
            if fa:
                break
        assert a.collect() == b.collect()
        assert a.get_calculated_checksum() == b.get_calculated_checksum()


def test_synthetic_configs_small(pkg, ctx, oracle, exec_mode):
    """Small instances of every BASELINE.json config against the oracle AND libzstd."""
    import datagen as G
    sets = [
        G.config_c2b(total_bytes=4 << 20, cache=False),
        G.config_c2a(total_bytes=2 << 20, nframes=2, cache=False),
        G.config_c3(nframes=24, cache=False),
        G.config_c4(nframes=6, cache=False),
        G.config_c5(nframes=300, cache=False),
    ]
    for fs in sets:
        D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict.tobytes()) if fs.raw_dict is not None else None
        out = np.zeros(fs.D + 16, dtype=np.uint8)
        res = pkg.decode_frames(ctx, fs.comp, fs.frames_io(), out, forced_dict=D)
        assert (res["status"] == 0).all(), (fs.name, res[res["status"] != 0][:3])
        assert (res["out_size"] == fs.out_size).all()
        assert np.array_equal(out[:fs.D], fs.plain), fs.name
        o_out, o_sz = oracle.bulk_decode(fs.comp, fs.src_off, fs.src_size, fs.out_off, fs.out_size,
                                         raw_dict=fs.raw_dict.tobytes() if fs.raw_dict is not None else None, nthreads=4)
        assert np.array_equal(o_out[:fs.D], out[:fs.D]) and (o_sz == fs.out_size).all()


def test_pipelined_one_shot_many_chunks(pkg, ctx, monkeypatch):
    """The host-to-host one-shot call overlaps planning / PCIe / kernels over several chunks of frames; force tiny chunks."""
    import datagen as G
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(1 << 20))
    fs = G.config_c3(nframes=200, cache=False)
    out = np.zeros(fs.D + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, fs.comp, fs.frames_io(), out)
    assert (res["status"] == 0).all() and (res["out_size"] == fs.out_size).all()
    assert np.array_equal(out[:fs.D], fs.plain)
    assert (res["bytes_read"] == fs.src_size).all() and (res["has_checksum"] == 1).all()
    # a broken frame in the middle fails alone
    comp = fs.comp.copy()
    comp[int(fs.src_off[77]) + 12] ^= 0xFF
    res = pkg.decode_frames(ctx, comp, fs.frames_io(), out)
    assert res[77]["status"] != 0 or not np.array_equal(out[fs.out_off[77]:fs.out_off[77] + fs.out_size[77]], fs.plain[fs.out_off[77]:fs.out_off[77] + fs.out_size[77]])
    ok = np.ones(fs.nframes, bool); ok[77] = False
    assert (res["status"][ok] == 0).all()


def test_irregular_huffman_split_matches_reference_semantics(pkg, ctx, oracle):
    """SURVEY App. B.3: ruzstd derives the 4 literal stream sizes from bit exhaustion, not from (n+3)/4, and only checks the total.
    A frame with an uneven split is rejected by libzstd but decodes under the reference's rules; the GPU fast path must notice and
    replay the block exactly.  Also: the same frame with one stream truncated must fail with the oracle's error."""
    import craft
    import datagen as G
    zo, bz = oracle.error_names(), pkg.error_names()
    for seed, shift in [(77, 7), (78, 1), (79, 250)]:
        text = G.gen_text(60000, seed)
        frame, plain = craft.irregular_huffman_split(oracle, G.compress(text), shift=shift)
        with pytest.raises(RuntimeError):
            G.decompress(frame, len(plain))            # the stock decoder refuses it
        exp, _ = oracle.decode_frame(frame)
        assert exp == plain
        out = np.zeros(len(plain) + 16, dtype=np.uint8)
        io = np.zeros(1, dtype=pkg.binding.FRAME_IO_DTYPE); io[0] = (0, len(frame), 0, len(plain))
        res = pkg.decode_frames(ctx, np.frombuffer(frame, dtype=np.uint8), io, out)
        assert res[0]["status"] == 0 and out[:len(plain)].tobytes() == plain
        dec = pkg.FrameDecoder(ctx)
        r = dec.reset(frame); dec.decode_blocks(r, pkg.ALL)
        assert dec.collect() == plain and dec.get_calculated_checksum() == dec.get_checksum_from_data()
        # corrupt the jump table: stream 1 one byte shorter, stream 2 one byte longer -> same error as the oracle
        bad = bytearray(frame)
        pos = frame.index(frame[:4]) + 0
        hdr_end, _ = craft._parse_single_block(frame)
        # literals header is 5 bytes (size format 3); jump table follows the tree description
        lit0 = hdr_end + 3 + 5
        tree = bad[lit0]
        tlen = 1 + (tree if tree < 128 else (tree - 127 + 1) // 2)
        j = lit0 + tlen
        v = int.from_bytes(bad[j:j + 2], "little") - 1
        bad[j:j + 2] = v.to_bytes(2, "little")
        bad = bytes(bad)
        try:
            e_out, _ = oracle.decode_frame(bad); e_err = None
        except oracle.OracleError as e:
            e_out, e_err = None, (zo[e.code].replace("ZO_", ""), e.stage)
        res = pkg.decode_frames(ctx, np.frombuffer(bad, dtype=np.uint8), io, out)
        if e_err is None:
            assert res[0]["status"] == 0 and out[:res[0]["out_size"]].tobytes() == e_out
        else:
            assert (bz[int(res[0]["status"])].replace("B200Z_", ""), int(res[0]["stage"])) == e_err


def test_target_too_small_and_capacity_isolation(pkg, ctx, exec_mode):
    """A frame that does not fit its out_cap fails alone and never writes past its slot (checked on the device buffer)."""
    import torch
    import datagen as G
    fs = G.config_c3(nframes=4, cache=False)
    io = fs.frames_io()
    io["out_cap"][2] = 1000
    d_out = torch.full((fs.D + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, fs.comp, io)
    b.run(d_out)
    res = b.finish()
    out = d_out.cpu().numpy()
    names = pkg.error_names()
    assert names[int(res[2]["status"])] == "B200Z_ERR_TARGET_TOO_SMALL"
    for i in (0, 1, 3):
        assert res[i]["status"] == 0
        assert np.array_equal(out[fs.out_off[i]:fs.out_off[i] + fs.out_size[i]], fs.plain[fs.out_off[i]:fs.out_off[i] + fs.out_size[i]])
    assert (out[int(fs.out_off[2]) + 1000:int(fs.out_off[3])] == 0xAB).all()
    assert (out[fs.D:] == 0xAB).all()


def test_truncation_sweep_matches_oracle(pkg, ctx, oracle, exec_mode):
    """Every prefix of a small frame: same outcome (bytes or error leaf + stage) as the oracle."""
    data = read_golden("decodecorpus", "z000002.zst")
    zo, bz = oracle.error_names(), pkg.error_names()
    cuts = list(range(0, min(len(data), 400))) + list(range(400, len(data), 97))
    frames = [data[:c] for c in cuts]
    io, comp, total = _io(pkg, frames, [1 << 16] * len(frames))
    out = np.zeros(total + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, comp if len(comp) else np.zeros(1, np.uint8), io, out)
    for i, f in enumerate(frames):
        try:
            exp, _ = oracle.decode_frame(f); err = None
        except oracle.OracleError as e:
            exp, err = None, (zo[e.code].replace("ZO_", ""), e.stage)
        if err is None:
            assert res[i]["status"] == 0 and out[io[i]["out_off"]:io[i]["out_off"] + res[i]["out_size"]].tobytes() == exp
        else:
            assert (bz[int(res[i]["status"])].replace("B200Z_", ""), int(res[i]["stage"])) == err, (cuts[i], res[i], err)


def test_bitflip_sweep_matches_oracle(pkg, ctx, oracle, exec_mode):
    """Single-bit corruptions of a compressed block: same outcome as the oracle, no device fault."""
    data = bytearray(read_golden("decodecorpus", "z000005.zst"))
    rng = np.random.Generator(np.random.PCG64(11))
    zo, bz = oracle.error_names(), pkg.error_names()
    frames = []
    for _ in range(300):
        d = bytearray(data)
        pos = int(rng.integers(4, len(d)))
        d[pos] ^= 1 << int(rng.integers(0, 8))
        frames.append(bytes(d))
    cap = 1 << 21
    io, comp, total = _io(pkg, frames, [cap] * len(frames))
    import torch
    d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    b = pkg.Batch(ctx, comp, io)
    b.run(d_out)
    res = b.finish()
    out = d_out.cpu().numpy()
    same = 0
    for i, f in enumerate(frames):
        try:
            exp, _ = oracle.decode_frame(f); err = None
        except oracle.OracleError as e:
            exp, err = None, (zo[e.code].replace("ZO_", ""), e.stage)
        if err is None:
            if len(exp) <= cap:
                assert res[i]["status"] == 0 and out[io[i]["out_off"]:io[i]["out_off"] + res[i]["out_size"]].tobytes() == exp, i
                same += 1
        else:
            assert (bz[int(res[i]["status"])].replace("B200Z_", ""), int(res[i]["stage"])) == err, (i, res[i], err)
    assert same > 0


def test_exec_run_shapes(pkg, ctx, oracle, exec_mode):
    """Sequence shapes that steer k_exec's batch paths: overlapping matches (offset < length, incl. offset 1), matches and literal
    runs far longer than a row, batches above the fast path's byte cap, odd sequence counts, repeat offsets after zero literal
    lengths.  Bit-exact against the plaintext and the oracle."""
    import datagen as G
    rng = np.random.Generator(np.random.PCG64(0xE8EC))
    def rnd(n): return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    text = G.gen_text(200000, 77).tobytes()
    pieces = [
        b"a" * 70000,                                                    # offset 1, length >> row: one long overlapping match
        (b"abc" * 9000) + rnd(100) + (b"xy" * 20000),                    # short periods
        rnd(3000) + b"\0" * 5000 + rnd(40) + b"\0" * 17 + rnd(9000),      # long literal runs around long matches
        b"".join(text[i * 97:i * 97 + 61] + b"=" * (i % 40) for i in range(1500)),   # text with runs of every length 0..39
        b"".join(rnd(700) + text[1000:1000 + 300 + i] for i in range(60)),           # ~1 KB per sequence: batches above the byte cap
        text[:131072],
        text[5000:5000 + 64 * 13 + 7],                                   # tiny frame, odd sequence count
        b"".join(text[200 * i:200 * i + 40] * 3 for i in range(400)),    # immediate repeats: repeat offsets with zero literal length
    ]
    frames = [G.compress(np.frombuffer(p, dtype=np.uint8)) for p in pieces]
    comp = np.frombuffer(b"".join(bytes(f) for f in frames), dtype=np.uint8)
    io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, (f, p) in enumerate(zip(frames, pieces)):
        io[i] = (so, len(f), oo, len(p))
        so += len(f); oo += len(p)
    out = np.zeros(oo + 16, dtype=np.uint8)
    res = pkg.decode_frames(ctx, comp, io, out)
    assert (res["status"] == 0).all(), res[res["status"] != 0][:3]
    plain = b"".join(pieces)
    for i, p in enumerate(pieces):
        got = out[io[i]["out_off"]:io[i]["out_off"] + len(p)].tobytes()
        assert got == p, f"piece {i}: GPU output differs from the plaintext"
        assert oracle.decode_frame(bytes(frames[i]))[0] == p
    assert (out[oo:] == 0).all()


def test_block_level_entry(pkg, ctx, oracle, manifest, exec_mode):
    """b200z_decode_blocks_batch: the thin FFI for a host that keeps the reference's own header parsing (replaces the call site
    BlockDecoder::decompress_block, block_decoder.rs:97-197).  Descriptors come from tests/refwalk.py (a restatement of the
    reference's header parsers); per-block output sizes are checked against the oracle's block trace, bytes against the corpus."""
    import refwalk
    B = pkg.binding
    names = sorted(manifest["corpus"])[:40]
    frames = [read_golden("decodecorpus", n) for n in names]
    sizes = [manifest["corpus"][n]["size"] for n in names]
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    comp, blocks, fr = refwalk.walk(frames, offs, sizes, (B.BLOCK_DESC_DTYPE, B.BLOCK_FRAME_DTYPE))
    out = np.zeros(int(sum(sizes)) + 16, dtype=np.uint8)
    st, fo = pkg.decode_blocks(ctx, blocks, fr, comp, out)
    assert (st["status"] == 0).all(), st[st["status"] != 0][:3]
    nb = 0
    for i, n in enumerate(names):
        assert fo[i] == sizes[i], n
        got = out[offs[i]:offs[i] + sizes[i]].tobytes()
        assert hashlib.sha256(got).hexdigest() == manifest["corpus"][n]["sha256"], n
        d = oracle.FrameDecoder(); d.trace_enable()
        r = d.reset(frames[i]); d.decode_blocks(r); d.collect()
        tblocks, _, _ = d.trace()
        assert len(tblocks) == fr[i]["num_blocks"]
        for k, tb in enumerate(tblocks):
            b = blocks[fr[i]["first_block"] + k]
            assert st[fr[i]["first_block"] + k]["out_size"] == tb["out_size"], (n, k)
            if tb["block_type"] == 2:
                assert (b["literals_type"], b["regenerated_size"], b["num_sequences"]) == (tb["literals_type"], tb["regenerated_size"], tb["num_sequences"])
            nb += 1
    assert nb > 300
    # device-resident input and output
    import torch
    d_in = torch.from_numpy(comp.copy()).cuda()
    d_out = torch.zeros(len(out), dtype=torch.uint8, device="cuda")
    st2, fo2 = pkg.decode_blocks(ctx, blocks, fr, d_in, d_out)
    assert (st2["status"] == 0).all() and np.array_equal(d_out.cpu().numpy()[:sum(sizes)], out[:sum(sizes)])
    # a corrupted block fails alone: its frame stops there, later blocks are "not reached", other frames are untouched
    bad = comp.copy()
    victim = next(j for j in range(len(blocks)) if blocks[j]["block_type"] == 2 and blocks[j]["num_sequences"] > 8 and not blocks[j]["last_block"])
    bad[int(blocks[victim]["src_off"]) + int(blocks[victim]["content_size"]) - 1] = 0   # sequence bitstream without its padding marker
    st3, fo3 = pkg.decode_blocks(ctx, blocks, fr, bad, np.zeros_like(out))
    fidx = next(i for i in range(len(fr)) if fr[i]["first_block"] <= victim < fr[i]["first_block"] + fr[i]["num_blocks"])
    assert st3[victim]["status"] > 0
    lo, hi = fr[fidx]["first_block"], fr[fidx]["first_block"] + fr[fidx]["num_blocks"]
    assert (st3[lo:victim]["status"] == 0).all() and (st3[victim + 1:hi]["status"] == B.BLOCK_NOT_REACHED).all()
    others = np.ones(len(st3), bool); others[lo:hi] = False
    assert (st3[others]["status"] == 0).all()
    # a descriptor that disagrees with the block content is rejected
    wrong = blocks.copy()
    wrong[victim]["num_sequences"] += 1
    with pytest.raises(pkg.B200ZError):
        pkg.decode_blocks(ctx, wrong, fr, comp, np.zeros_like(out))


@pytest.mark.slow
@pytest.mark.parametrize("config", ["c2a", "c3", "c4", "c5"])
def test_full_size_configs(pkg, ctx, config):
    """The other BASELINE.json configs at their FULL sizes (C2a: one chained 1 GiB frame of 8192 blocks; C3: 10,000 x 64 KiB;
    C4: 4096 x 1 MiB Silesia-mix frames; C5: 100,000 small frames + a 110 KiB raw-content dictionary): every frame succeeds,
    sizes match and the plaintext is the generator's, byte for byte (size-independent check; small instances of the same
    configs are compared with the oracle in test_synthetic_configs_small)."""
    import torch
    import datagen as G
    fs = {"c2a": lambda: G.config_c2a(total_bytes=1 << 30, nframes=1, cache=False), "c3": lambda: G.config_c3(nframes=10000, cache=False),
          "c4": lambda: G.config_c4(nframes=4096, cache=False), "c5": lambda: G.config_c5(nframes=100000, cache=False)}[config]()
    D = pkg.Dictionary.raw_content(ctx, 1, fs.raw_dict.tobytes()) if fs.raw_dict is not None else None
    b = pkg.Batch(ctx, fs.comp, fs.frames_io(), forced_dict=D)
    d_out = torch.zeros(fs.D + 64, dtype=torch.uint8, device="cuda")
    b.run(d_out)
    res = b.finish()
    assert (res["status"] == 0).all(), (config, res[res["status"] != 0][:3])
    assert (res["out_size"] == fs.out_size).all() and (res["bytes_read"] == fs.src_size).all()
    got = d_out[:fs.D].cpu().numpy()
    assert np.array_equal(got, fs.plain), config
    b.close()


def test_exact_path_replay_rolls_back(pkg, ctx, oracle, monkeypatch):
    """k_exec (one warp per frame) consumes a block's sequences while k_fse is still decoding it; when k_fse's fast path gives the
    block up late (here: thousands of ordinary text sequences, then one sequence with more than 32 extra bits -- a far offset with
    a long literal run and a long match) its exact path rewrites the records with raw offsets, and k_exec must roll the block back
    and run it again.  Large-window frames; all frames forced onto the warp kernel."""
    import datagen as G
    monkeypatch.setenv("B200Z_EXEC_MODE", "warp")
    rng = np.random.Generator(np.random.PCG64(77))
    pieces = []
    for i in range(24):
        far = rng.integers(0, 256, 2 << 20, dtype=np.uint8)
        text = G.gen_text(100000 + 1000 * i, 500 + i)
        fresh = rng.integers(0, 256, 20000 + 37 * i, dtype=np.uint8)
        pieces.append(np.concatenate([far, text, fresh, far[5000:5000 + 9000 + 11 * i]]))
    frames = [G.compress(p_, level=3, window_log=22) for p_ in pieces]
    io, comp, total = _io(pkg, frames, [len(p_) for p_ in pieces])
    import torch
    b = pkg.Batch(ctx, comp, io)
    d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        b.run(d_out)
        res = b.finish()
        assert (res["status"] == 0).all(), res[res["status"] != 0][:3]
        out = d_out.cpu().numpy()
        for i, p_ in enumerate(pieces):
            assert np.array_equal(out[io[i]["out_off"]:io[i]["out_off"] + len(p_)], p_), i
    # the exact path really was taken for blocks with many sequences (raw-offset flag), otherwise this test does not test what it says
    nblocks = b.info()["blocks"]
    raw_big = [k for k in range(nblocks) if (b.debug_block_flags(k) & 1) and len(b.debug_sequences(k)) > 1000]
    assert len(raw_big) >= 4, "no long block went through k_fse's exact path"
    b.close()


def test_device_walk_matches_host_plan(pkg, ctx, oracle, manifest):
    """Device-resident input: k_walk follows the frame / block / section headers on the GPU and the planner works from its digests
    (no copy of the compressed data back to the host).  Every outcome -- status, stage, sizes, bytes read, checksum, plaintext --
    must equal what the host walk produces from the same bytes given as host input: the golden corpus, every fuzz artifact (incl.
    the ones without a dictionary id), truncated frames, garbage."""
    import torch
    frames = [read_golden("decodecorpus", n) for n in sorted(manifest["corpus"])]
    for sub, files in manifest["fuzz"].items():
        frames += [read_golden("fuzz", sub, f) for f in files]
    data = read_golden("decodecorpus", "z000002.zst")
    frames += [data[:c] for c in list(range(0, 40)) + list(range(40, len(data), 53))]
    rng = np.random.Generator(np.random.PCG64(3))
    frames += [bytes([0x28, 0xB5, 0x2F, 0xFD]) + rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in rng.integers(0, 300, 40)]
    frames = [f if len(f) else b"" for f in frames]
    caps = [1 << 17] * len(frames)
    for i, n in enumerate(sorted(manifest["corpus"])):
        caps[i] = manifest["corpus"][n]["size"]
    io, comp, total = _io(pkg, frames, caps)
    comp = comp if len(comp) else np.zeros(1, np.uint8)
    outs = {}
    for mode, src in (("host", comp), ("device", torch.from_numpy(comp.copy()).cuda())):
        d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
        b = pkg.Batch(ctx, src, io)
        b.run(d_out)
        outs[mode] = (b.finish().copy(), d_out.cpu().numpy(), b.info()["blocks"])
        b.close()
    rh, oh, nbh = outs["host"]
    rd, od, nbd = outs["device"]
    assert nbh == nbd and nbd > 2000
    for k in rh.dtype.names:
        assert np.array_equal(rh[k], rd[k]), k
    assert np.array_equal(oh, od)
    assert (rd["status"] == 0).sum() >= 101 and (rd["status"] != 0).sum() > 50
