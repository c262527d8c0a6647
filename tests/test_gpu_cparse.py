"""The compressor on the GPU against the plain model of its parse (tests/cparse.py): every Compressed block's literals and
sequences (through the oracle's trace) are the model's, and every frame is reference_frame's byte for byte -- which also pins the
Raw blocks' parse, k_cenc's 32-lane encode_block against the 1-lane host build, k_cassemble's layout and k_cxxh64 -- in one
submission, one frame per submission, from host and device memory, against raw-content and formatted dictionaries with and without
their tables.  The frame checks take the level; test_gpu_clazy.py runs them at LAZY (tests/clazy.py).  The dictionary finalizer's
statistics are the model's counts, and both checksum kernels (k_cxxh64, k_xxh64) equal the plain XXH64 at the lengths where their
stripe loops change shape, at every address residue mod 8."""
import ctypes as C
import struct

import numpy as np
import pytest

import clazy
import cparse
import datagen
from conftest import read_golden

pytestmark = pytest.mark.gpu

LEVELS = {"fastest": (cparse.FASTEST, cparse.cases()), "lazy": (clazy.LAZY, clazy.cases())}
CASES = LEVELS["fastest"][1]
PLAIN = [c for c in CASES if c.content is None]
WITH_DICT = [c for c in CASES if c.content is not None]

_models, _refs = {}, {}


def model(name, c):
    """The parse of case c at the level, computed once."""
    if (name, c.id) not in _models:
        _models[name, c.id] = cparse.parse(c.frames, c.content, LEVELS[name][0])
    return _models[name, c.id]


def reference(name, c, i, **kw):
    """reference_frame of frame i of case c at the level, cached per options."""
    key = (name, c.id, i, tuple(sorted((k, v if not isinstance(v, bytes) else hash(v)) for k, v in kw.items())))
    if key not in _refs:
        _refs[key] = cparse.reference_frame(c.frames[i], model(name, c)[i], level=LEVELS[name][0], **kw)
    return _refs[key]


def compress(pkg, ctx, datas, dict=None, dict_tables=False, device=False, level=1, checksum=True, window_log=cparse.WINDOW_LOG_MIN):
    """compress_frames over datas laid out back to back at window_log; returns the frames and the result rows."""
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    parts = []
    for i, d in enumerate(datas):
        parts.append(d)
        cap = pkg.compress_bound(len(d), dict)
        io[i] = (so, len(d), oo, cap)
        so += len(d)
        oo += cap
    src = np.frombuffer(b"".join(parts), dtype=np.uint8) if so else np.zeros(1, dtype=np.uint8)
    out = np.zeros(max(oo, 1), dtype=np.uint8)
    if device:
        import torch
        src_t, out_t = torch.from_numpy(src.copy()).cuda(), torch.zeros(out.size, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, src_t, io, out_t, level, checksum, dict=dict, dict_tables=dict_tables, window_log=window_log)
        out = out_t.cpu().numpy()
    else:
        res = pkg.compress_frames(ctx, src, io, out, level, checksum, dict=dict, dict_tables=dict_tables, window_log=window_log)
    assert (res["status"] == 0).all()
    return [out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(datas))], res


def traced_blocks(oracle, f, content=None, formatted=None):
    """Per block of frame f, decoded by the oracle: (block type, literals, [(ll, ml, actual offset), ...])."""
    d = oracle.FrameDecoder()
    d.trace_enable()
    if formatted is not None:
        d.add_dict(formatted)
    if content is not None:
        d.add_raw_content_dict(1, content)
    r = d.reset(f)
    if content is not None:
        d.force_dict(1)
    d.decode_blocks(r)
    d.collect()
    blocks, lits, seqs = d.trace()
    out = []
    for b in blocks:
        lo, k = int(b["lit_offset"]), int(b["seq_offset"])
        s = [(int(ll), int(ml), int(off)) for ll, ml, _, off in seqs[k:k + int(b["num_sequences"])].tolist()]
        out.append((int(b["block_type"]), lits[lo:lo + int(b["regenerated_size"])], s))
    return out


def check_parse(c, blocks, frames, oracle, content=None, formatted=None):
    """Every Compressed block of the GPU's frames of case c has the literals and sequences of `blocks`, the model's parse."""
    for i, f in enumerate(frames):
        want = blocks[i]
        got = traced_blocks(oracle, f, content, formatted)
        assert len(got) == len(want), (c.id, i)
        for k, ((btype, lits, seqs), w) in enumerate(zip(got, want)):
            if btype == 1:
                assert w[0] == "rle", f"{c.id} frame {i} block {k}: RLE on the GPU, {len(w[1])} sequences in the model"
            elif btype == 2:
                assert w[0] != "rle", f"{c.id} frame {i} block {k}: Compressed on the GPU, RLE in the model"
                if seqs != w[1]:
                    j = next((j for j, (a, b) in enumerate(zip(seqs, w[1])) if a != b), min(len(seqs), len(w[1])))
                    pytest.fail(f"{c.id} frame {i} block {k}: sequence {j} differs: GPU "
                                f"{seqs[j] if j < len(seqs) else None}, model {w[1][j] if j < len(w[1]) else None} "
                                f"({len(seqs)} vs {len(w[1])} sequences)")
                assert lits == w[0], f"{c.id} frame {i} block {k}: literals differ"


def test_parse_is_the_models(pkg, ctx, oracle):
    frames, _ = compress(pkg, ctx, [f for c in PLAIN for f in c.frames])
    at = 0
    for c in PLAIN:
        check_parse(c, model("fastest", c), frames[at:at + len(c.frames)], oracle)
        at += len(c.frames)
    for c in WITH_DICT:
        D = pkg.Dictionary.raw_content(ctx, 1, c.content)
        frames, _ = compress(pkg, ctx, c.frames, dict=D)
        check_parse(c, model("fastest", c), frames, oracle, content=c.content)


def check_reference_frames(pkg, ctx, name):
    """The frames of every case without a dictionary at the level (LEVELS) are reference_frame's: in one submission, and one
    frame per submission from host and device memory."""
    level = getattr(pkg, name.upper())
    plain = [c for c in LEVELS[name][1] if c.content is None]
    frames, _ = compress(pkg, ctx, [f for c in plain for f in c.frames], level=level)
    at = 0
    for c in plain:
        for i in range(len(c.frames)):
            assert frames[at + i] == reference(name, c, i), f"{c.id} frame {i}"
        at += len(c.frames)
    for c in plain:                                                     # one frame per submission, host and device
        for i, data in enumerate(c.frames):
            for device in (False, True):
                assert compress(pkg, ctx, [data], device=device, level=level)[0][0] == reference(name, c, i), \
                    f"{c.id} frame {i} device={device}"


def check_reference_frames_with_dictionaries(pkg, ctx, name):
    """The frames of every case with a dictionary at the level (LEVELS) are reference_frame's: against its raw content from host
    and device memory, and against the finalized dictionary with and without its tables."""
    level = getattr(pkg, name.upper())
    for c in [c for c in LEVELS[name][1] if c.content is not None]:
        R = pkg.Dictionary.raw_content(ctx, 1, c.content)
        for device in (False, True):
            frames, _ = compress(pkg, ctx, c.frames, dict=R, device=device, level=level)
            for i, f in enumerate(frames):
                assert f == reference(name, c, i), f"{c.id} frame {i} raw content device={device}"
        if len(c.content) < 8:                                           # the finalizer's smallest content
            continue
        fin = pkg.finalize_dict(ctx, c.content, c.frames[:50])
        assert fin.endswith(c.content)
        F = pkg.Dictionary.decode_dict(ctx, fin)
        for tables in (False, True):
            frames, _ = compress(pkg, ctx, c.frames, dict=F, dict_tables=tables, level=level)
            for i, f in enumerate(frames):
                want = reference(name, c, i, dict_id=F.id, dict_tables=fin if tables else None)
                assert f == want, f"{c.id} frame {i} finalized dictionary tables={tables}"


def test_frames_are_the_reference(pkg, ctx):
    check_reference_frames(pkg, ctx, "fastest")


def test_frames_with_dictionaries_are_the_reference(pkg, ctx):
    check_reference_frames_with_dictionaries(pkg, ctx, "fastest")


def test_golden_formatted_dictionary(pkg, ctx, oracle, manifest):
    dic = read_golden("dict_tests", "dictionary")
    did, offs, n = C.c_uint32(), (C.c_uint32 * 3)(), C.c_size_t()
    assert oracle.lib().zo_kat_decode_dict(dic, len(dic), C.byref(did), offs, C.byref(n)) == 0
    content = dic[len(dic) - n.value:]
    names = sorted(manifest["dict"])[:40]
    datas = [oracle.decode_frame(read_golden("dict_tests", "files", x), dict_raw=dic)[0] for x in names]
    datas.append(content[-3000:-1000] + content[-64:] + bytes(range(256)))
    c = cparse.Case("golden", "dict_tests-dictionary", datas, content)
    blocks = cparse.parse(c.frames, content)
    D = pkg.Dictionary.decode_dict(ctx, dic)
    assert D.id == did.value and D.content_size == len(content)
    for tables in (False, True):
        frames, _ = compress(pkg, ctx, datas, dict=D, dict_tables=tables)
        check_parse(c, blocks, frames, oracle, formatted=dic)
        for i, f in enumerate(frames):
            assert f == cparse.reference_frame(datas[i], blocks[i], dict_id=D.id, dict_tables=dic if tables else None), \
                f"{names[i] if i < len(names) else 'crafted'} tables={tables}"


def test_finalizer_statistics_are_the_models_counts(pkg, ctx):
    """finalize_dict's statistics are the model's counts over more than one DS_BLOCKS submission: C5 pieces, random samples the
    encoder would write Raw (still counted), empty and RLE samples (not), and samples over 128 KiB (their first block only)."""
    fs = datagen.config_c5(nframes=1900, cache=False)
    plain = fs.plain.tobytes()
    content = fs.raw_dict.tobytes()
    samples = [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)]
    rng = np.random.default_rng(11)
    samples += [rng.integers(0, 256, int(rng.integers(1, 3000)), dtype=np.uint8).tobytes() for _ in range(150)]
    samples += [b""] * 5 + [b"\x07" * 9000, content[-6000:]]
    samples += [bytes(datagen.gen_text(200000, 12)), rng.integers(0, 256, 140000, dtype=np.uint8).tobytes(), b"r" * 140000]
    rng.shuffle(samples)
    assert len(samples) > cparse.DS_BLOCKS
    want = pkg.dict_from_counts(cparse.counts(samples, content), content)
    before = ctx.kernel_launches()
    assert pkg.finalize_dict(ctx, content, samples) == want
    assert ctx.kernel_launches() - before == 1 + 2 * -(-len(samples) // cparse.DS_BLOCKS)


LENGTHS = list(range(41)) + sorted({32 * m + r for m in (15, 16, 17, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025) for r in (0, 7, 31)})


def test_checksums_at_every_residue(pkg, ctx):
    """k_cxxh64 (Uncompressed-level frames, input at every residue mod 8: the aligned 32-stripe pipeline and the unaligned
    16-stripe batches) and k_xxh64 (those frames decoded with FLAG_CHECKSUM, output at every residue mod 8) against the plain
    XXH64."""
    rng = np.random.default_rng(13)
    datas = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in LENGTHS]
    want = [cparse.xxh64(d) & 0xFFFFFFFF for d in datas]
    dec = pkg.Context(0)
    dec.set_flags(pkg.binding.FLAG_CHECKSUM)
    try:
        for r in range(8):
            for device in (False, True):
                frames, res = compress_at(pkg, ctx, datas, r, device)
                for n, d, f, x, w in zip(LENGTHS, datas, frames, res, want):
                    assert x["checksum"] == w and struct.unpack("<I", f[-4:])[0] == w, (n, r, device)
                    assert f == cparse.reference_frame(d, [None] * max(1, -(-n // cparse.BLOCK)), level=cparse.UNCOMPRESSED), (n, r)
            io = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
            so = oo = 0
            for i, (f, d) in enumerate(zip(frames, datas)):
                oo += (r - oo) % 8
                io[i] = (so, len(f), oo, len(d))
                so += len(f)
                oo += len(d)
            out = np.zeros(oo + 16, dtype=np.uint8)
            res = pkg.decode_frames(dec, np.frombuffer(b"".join(frames), dtype=np.uint8), io, out)
            for i, (n, w) in enumerate(zip(LENGTHS, want)):
                assert res[i]["status"] == 0 and res[i]["has_calculated_checksum"] == 1, (n, r)
                assert res[i]["calculated_checksum"] == w == res[i]["checksum_from_data"], (n, r)
                assert out[io[i]["out_off"]:io[i]["out_off"] + n].tobytes() == datas[i]
    finally:
        dec.close()


def compress_at(pkg, ctx, datas, r, device):
    """Uncompressed-level frames of datas, every input starting at an offset = r mod 8."""
    io = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    buf = bytearray()
    oo = 0
    for i, d in enumerate(datas):
        buf += b"\0" * ((r - len(buf)) % 8)
        cap = pkg.compress_bound(len(d))
        io[i] = (len(buf), len(d), oo, cap)
        buf += d
        oo += cap
    src = np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8)
    out = np.zeros(oo, dtype=np.uint8)
    if device:
        import torch
        out_t = torch.zeros(out.size, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, torch.from_numpy(src.copy()).cuda(), io, out_t, 0, True)
        out = out_t.cpu().numpy()
    else:
        res = pkg.compress_frames(ctx, src, io, out, 0, True)
    assert (res["status"] == 0).all()
    return [out[io[i]["dst_off"]:io[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(datas))], res
