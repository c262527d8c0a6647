"""The raw-content dictionary trainer on the GPU (b200z_dict_train_raw): byte-exact against the NumPy model (tests/dicttrain.py)
with its segment table, deterministic across inputs in host or device memory, runs and contexts, usable by this library's
compressor and decoders and by libzstd, at least as good as the quality floors below, and rejecting bad arguments before any
launch."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

import datagen
import dicttrain as M
from conftest import ROOT

gpu = pytest.mark.gpu
DICT = 112640


@pytest.fixture(scope="module")
def c5():
    """C5 frames 0-3999: plaintext pieces (0-1999 train, 2000-3999 are held out)."""
    fs = datagen.config_c5(nframes=4000, cache=False)
    plain = fs.plain.tobytes()
    return [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)]


def same_as_model(pkg, ctx, data, dict_size, sizes=None, seg=2048):
    got, segs = pkg.create_raw_dict(ctx, data, dict_size, sample_sizes=sizes, segment_size=seg, segments=True)
    want, wsegs = M.train(data, dict_size, sizes, seg)
    assert [(int(s["epoch"]), int(s["src_off"]), int(s["size"]), int(s["score"])) for s in segs] == wsegs
    assert got == want, (len(got), len(want))
    return got


def text(n, seed):
    return bytes(datagen.gen_text(n, seed)) if n else b""


@gpu
@pytest.mark.parametrize("seg", [2048, 512, 256])
def test_c5_samples_match_model(pkg, ctx, c5, seg):
    train = c5[:2000]
    d = same_as_model(pkg, ctx, b"".join(train), DICT, [len(p) for p in train], seg)
    assert len(d) == DICT


@gpu
@pytest.mark.parametrize("kind", ["c2b_text", "silesia_mix"])
def test_8mib_one_sample_matches_model(pkg, ctx, kind):
    data = datagen.c2_text_plain(8 << 20, seed=0xE90001).tobytes() if kind == "c2b_text" else datagen.gen_silesia_mix(8 << 20, 0xC40007).tobytes()
    same_as_model(pkg, ctx, data, DICT)


@gpu
def test_all_zero_input(pkg, ctx):
    d = same_as_model(pkg, ctx, bytes(1 << 20), DICT)
    assert d == bytes(DICT)


@gpu
@pytest.mark.parametrize("n", [16, 17, 2047, 2048, 2049, 9999, 10000, 10001, 20000])
def test_sizes_around_the_epoch_rule(pkg, ctx, n):
    data = text(n, 100 + n)
    for dict_size in (DICT, 4096, 100):
        same_as_model(pkg, ctx, data, dict_size)


@gpu
def test_samples_shorter_than_a_kmer(pkg, ctx):
    data = text(21000, 5)
    same_as_model(pkg, ctx, data[:20000], DICT, [10, 15, 1, 0, 14] * 500)
    d, segs = pkg.create_raw_dict(ctx, data, DICT, [7] * 3000, segments=True)
    assert same_as_model(pkg, ctx, data, DICT, [7] * 3000) == d
    # no k-mer anywhere: each of the two epochs takes its first segment, with score 0
    assert segs["src_off"].tolist() == [0, 10000] and segs["score"].tolist() == [0, 0] and d == data[:2048] + data[10000:12048]


@gpu
@pytest.mark.parametrize("seg", [16, 256, 2048, 65536])
def test_segment_sizes(pkg, ctx, seg):
    data = text(300_000, 7)
    sizes = [1000 + (i % 7) * 500 for i in range(80)]
    sizes.append(len(data) - sum(sizes))
    same_as_model(pkg, ctx, data, DICT, None, seg)
    same_as_model(pkg, ctx, data, 20000, sizes, seg)


@gpu
def test_dictionary_sizes(pkg, ctx):
    data = text(50_000, 9)
    for L in (2048, 256):
        for dict_size in (0, 100, L - 1, L, DICT, len(data) + 1, 10 * len(data)):
            d = same_as_model(pkg, ctx, data, dict_size, None, L)
            assert len(d) <= dict_size


@gpu
def test_host_device_runs_and_contexts_agree(pkg, ctx, c5):
    import torch
    train = c5[:500]
    data, sizes = b"".join(train), [len(p) for p in train]
    a = pkg.create_raw_dict(ctx, data, DICT, sizes, segments=True)
    b = pkg.create_raw_dict(ctx, torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(), DICT, sizes, segments=True)
    c = pkg.create_raw_dict(ctx, data, DICT, sizes, segments=True)
    other = pkg.Context(0)
    d = pkg.create_raw_dict(other, data, DICT, sizes, segments=True)
    other.close()
    for x in (b, c, d):
        assert x[0] == a[0] and (x[1] == a[1]).all()
    assert pkg.create_raw_dict(ctx, train, DICT) == a[0]   # a list of samples


@gpu
def test_reference_names(pkg, ctx, c5, tmp_path):
    data = b"".join(c5[:300])
    want = pkg.create_raw_dict(ctx, data, 8192)
    out = io.BytesIO()
    pkg.create_raw_dict_from_source(ctx, io.BytesIO(data), len(data), out, 8192)
    assert out.getvalue() == want
    out = io.BytesIO()
    pkg.create_raw_dict_from_source(ctx, b"short", 5, out, 8192)
    assert out.getvalue() == b"short"
    paths = []
    for i, p in enumerate(c5[:40]):
        sub = tmp_path / f"d{i % 3}"
        sub.mkdir(exist_ok=True)
        paths.append(str(sub / f"f{i:03d}"))
        open(paths[-1], "wb").write(p)
    out = io.BytesIO()
    pkg.create_raw_dict_from_dir(ctx, str(tmp_path), out, 8192)
    order = sorted(range(40), key=lambda i: paths[i])
    assert out.getvalue() == pkg.create_raw_dict(ctx, [c5[i] for i in order], 8192)


def ratio_libzstd(pieces, content):
    return sum(len(p) for p in pieces) / sum(len(datagen.compress(p, level=3, raw_dict=content)) for p in pieces)


def zdict_train_content(pieces, cap):
    """ZDICT_trainFromBuffer's dictionary without its header (ZDICT_getDictHeaderSize): its content part."""
    z = datagen.zstd()
    z.ZDICT_trainFromBuffer.restype = C.c_size_t
    z.ZDICT_trainFromBuffer.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint]
    z.ZDICT_getDictHeaderSize.restype = C.c_size_t
    z.ZDICT_getDictHeaderSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZDICT_isError.restype = C.c_uint
    z.ZDICT_isError.argtypes = [C.c_size_t]
    buf = np.frombuffer(b"".join(pieces), dtype=np.uint8)
    sizes = np.array([len(p) for p in pieces], dtype=np.uintp)
    out = np.zeros(cap, dtype=np.uint8)
    n = z.ZDICT_trainFromBuffer(out.ctypes.data, cap, buf.ctypes.data, sizes.ctypes.data, len(pieces))
    assert not z.ZDICT_isError(n)
    h = z.ZDICT_getDictHeaderSize(out.ctypes.data, n)
    assert not z.ZDICT_isError(h)
    return out[h:n].tobytes()


@gpu
def test_quality_floors(pkg, ctx, c5):
    from test_compress_dict import compress_many
    train, held = c5[:2000], c5[2000:4000]
    sizes = [len(p) for p in train]
    d2048 = pkg.create_raw_dict(ctx, train, DICT)
    d256 = pkg.create_raw_dict(ctx, train, DICT, segment_size=256)
    r2048, r256 = ratio_libzstd(held, d2048), ratio_libzstd(held, d256)
    rz = ratio_libzstd(held, zdict_train_content(train, DICT))
    D = pkg.Dictionary.raw_content(ctx, 1, d2048)
    total = sum(len(p) for p in held)
    own = total / sum(len(f) for f in compress_many(pkg, ctx, held, dict=D, checksum=False)[0])
    own_none = total / sum(len(f) for f in compress_many(pkg, ctx, held, checksum=False)[0])
    print(f"held-out C5 ratio, libzstd level 3 + raw dictionary: L=2048 {r2048:.3f}, L=256 {r256:.3f}, "
          f"ZDICT_trainFromBuffer content {rz:.3f}; this library's compressor: {own:.3f} with L=2048, {own_none:.3f} without")
    assert len(d2048) == DICT and sum(sizes) > DICT
    assert r2048 >= 7.0
    assert r256 >= 9.0 and r256 >= rz
    assert own >= 3 * own_none


@gpu
def test_round_trip_through_compressor_and_decoders(pkg, ctx, c5):
    from test_compress_dict import batch_decode, compress_many
    d = pkg.create_raw_dict(ctx, c5[:2000], DICT)
    D = pkg.Dictionary.raw_content(ctx, 1, d)
    held = c5[2000:2300]
    frames, res = compress_many(pkg, ctx, held, dict=D)
    batch_decode(pkg, ctx, held, frames, forced=D)
    for p, f in zip(held, frames):
        assert datagen.decompress(f, len(p), raw_dict=d) == p


@gpu
def test_rejections_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    data = np.frombuffer(text(50_000, 11), dtype=np.uint8)
    out = np.zeros(DICT, dtype=np.uint8)
    segs = np.zeros(16, dtype=pkg.binding.DICT_SEGMENT_DTYPE)
    dlen, nseg = C.c_size_t(), C.c_size_t()

    def call(n=data.size, sizes=None, dict_size=8192, seg=2048, cap=DICT, segs_cap=16, with_segs=True):
        sz = None if sizes is None else np.array(sizes, dtype=np.uint64)
        return L.b200z_dict_train_raw(ctx.h, data.ctypes.data, n, 0, None if sz is None else sz.ctypes.data, 0 if sz is None else len(sz), dict_size,
                                      seg, out.ctypes.data, cap, C.byref(dlen), segs.ctypes.data if with_segs else None, segs_cap, C.byref(nseg))

    E = len(M.epochs(data.size, 8192, 2048))
    assert E == 4
    before = ctx.kernel_launches()
    bad = err["B200Z_ERR_INVALID_ARGUMENT"]
    assert call(seg=15) == bad and call(seg=65537) == bad
    assert call(sizes=[1000, data.size - 1001]) == bad and call(sizes=[1000, data.size - 999]) == bad
    assert call(n=1 << 32) == bad
    assert call(cap=8191) == bad
    assert call(dict_size=100, cap=99) == bad
    assert call(n=10, cap=9) == bad
    assert call(segs_cap=E - 1) == bad
    assert ctx.kernel_launches() == before
    assert call(segs_cap=E - 1, with_segs=False) == 0 and dlen.value == 8192
    assert ctx.kernel_launches() == before + 2 + E   # k_dtcount, k_dtprev and one k_dtepoch per epoch
    assert call(cap=8192, segs_cap=E) == 0 and nseg.value == E
    launches = ctx.kernel_launches()
    assert call(n=10, cap=10) == 0 and dlen.value == 10 and out[:10].tobytes() == data[:10].tobytes()
    assert call(dict_size=0, cap=0) == 0 and dlen.value == 0 and nseg.value == 0
    assert ctx.kernel_launches() == launches          # nothing to train: no launch


@gpu
def test_exact_need_is_accepted(pkg, ctx):
    """dict_cap and segments_cap equal to what the trainer writes are enough, one less is not; including an epoch shorter than L,
    where the need is below E * L."""
    L = pkg.lib()
    bad = {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_INVALID_ARGUMENT"]
    dlen, nseg = C.c_size_t(), C.c_size_t()
    for n, dict_size, seg in ((30_000, 200_000, 65536), (50_000, 8192, 2048), (50_000, 5000, 2048), (20_001, 112640, 256)):
        data = np.frombuffer(text(n, 13), dtype=np.uint8)
        ep = M.epochs(n, dict_size, seg)
        need = min(dict_size, sum(le for _, _, le in ep))
        out = np.zeros(need, dtype=np.uint8)
        segs = np.zeros(len(ep), dtype=pkg.binding.DICT_SEGMENT_DTYPE)

        def call(cap, scap):
            return L.b200z_dict_train_raw(ctx.h, data.ctypes.data, n, 0, None, 0, dict_size, seg, out.ctypes.data, cap, C.byref(dlen),
                                          segs.ctypes.data, scap, C.byref(nseg))
        assert call(need - 1, len(ep)) == bad and call(need, len(ep) - 1) == bad
        assert call(need, len(ep)) == 0 and dlen.value == need and nseg.value == len(ep)
        assert out.tobytes() == M.train(data.tobytes(), dict_size, None, seg)[0]


@gpu
def test_collection_at_the_top_of_the_size_range(pkg):
    """n = 2^32 - 1, the largest accepted size, in 6 epochs: the last CTA of the last epoch scores starts up to n - 2048, and its
    positions run to n - 16.  The input is zeros with 2,600 random bytes at the end, so the expected result follows without the
    model: epoch 0 takes the zeros at 0, epochs 1-4 find nothing left (score 0, first start), and epoch 5's best start, computed
    here by brute force over the tail, lies in that last tile."""
    import torch
    n, T, dict_size = (1 << 32) - 1, 2600, 6 * 2048
    ep = M.epochs(n, dict_size, 2048)
    assert len(ep) == 6
    e0, e1, le = ep[-1]
    s0 = e0 + (e1 - le - e0) // 4096 * 4096        # first start of the last tile of k_dtepoch (4096 starts per CTA)
    assert s0 + 4095 >= 1 << 32 and n - 16 + 512 >= 1 << 32
    tail = np.random.default_rng(17).integers(0, 256, T, dtype=np.uint8)
    Cn = T + 4200                                  # every position whose k-mer is not all zeros lies in this chunk
    chunk = np.zeros(Cn, dtype=np.uint8)
    chunk[-T:] = tail
    sl = M.slots(chunk.tobytes())
    zslot = M.slots(bytes(16))[0]
    valid = sl != M.NO_SLOT
    freq = np.bincount(sl[valid], minlength=1 << M.F)
    score0 = (n - Cn) + int(freq[zslot])
    freq[zslot] = 0                                # zeroed by epoch 0's segment
    W = 2048 - 15
    best, best_score = None, -1
    for i in range(Cn - 2048 + 1):
        w = sl[i:i + W]
        w = np.unique(w[w != M.NO_SLOT])
        sc = int(freq[w].sum())
        if sc > best_score:
            best, best_score = n - Cn + i, sc
    assert best >= s0 and best_score > 0
    ctx2 = pkg.Context(0)                          # its 28 GB of scratch goes with it
    try:
        d = torch.zeros(n, dtype=torch.uint8, device="cuda")
        d[n - T:] = torch.from_numpy(tail).cuda()
        before = ctx2.kernel_launches()
        got, segs = pkg.create_raw_dict(ctx2, d, dict_size, segments=True)
        assert ctx2.kernel_launches() - before == 2 + 6
        del d
    finally:
        ctx2.close()
        torch.cuda.empty_cache()
    want = [(0, 0, 2048, score0)] + [(e, ep[e][0], 2048, 0) for e in range(1, 5)] + [(5, best, 2048, best_score)]
    assert [(int(s["epoch"]), int(s["src_off"]), int(s["size"]), int(s["score"])) for s in segs] == want
    assert got == bytes(4 * 2048) + chunk[best - (n - Cn):best - (n - Cn) + 2048].tobytes() + bytes(2048)


def test_segment_struct_matches_the_binding(pkg, tmp_path):
    dt = pkg.binding.DICT_SEGMENT_DTYPE
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200zstd.h"', 'int main(void) {',
             '  printf("* %zu 0\\n", sizeof(b200z_dict_segment));']
    lines += [f'  printf("{f} %zu %zu\\n", offsetof(b200z_dict_segment, {f}), sizeof(((b200z_dict_segment *)0)->{f}));' for f in dt.names]
    lines += ['  return 0;', '}']
    src = tmp_path / "seg.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "seg"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    rows = [ln.split() for ln in subprocess.check_output([str(exe)]).decode().split("\n") if ln]
    assert rows[0] == ["*", str(dt.itemsize), "0"]
    for f, off, size in rows[1:]:
        assert dt.fields[f][1] == int(off) and dt.fields[f][0].itemsize == int(size), f
    assert len(rows) == 1 + len(dt.names)
