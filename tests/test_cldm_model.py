"""The long-distance match model (tests/cldm.py) on the CPU: its frames decode to their input with libzstd and the oracle within their
own Window_Descriptor, its anchors are content-defined and sparse, its kept matches obey the rule, the hand-computed edges hold,
and the host build of the header writer follows the Window_Descriptor rule."""
import os
import subprocess

import numpy as np
import pytest

import clazy
import cldm
import cparse
import datagen
import seqcraft

BLOCK = cldm.BLOCK


def planted(n, repeats, seed):
    """n random bytes with, for each (dst, src, length), data[dst:dst + length] = data[src:src + length]."""
    buf = bytearray(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())
    for dst, src, ln in repeats:
        buf[dst:dst + ln] = buf[src:src + ln]
    return bytes(buf)


def decode_checked(oracle, frame, data, window_log):
    """Decodes `frame` with the oracle (through its trace: the window is 2^window_log and every offset within it) and libzstd."""
    d = oracle.FrameDecoder()
    d.set_max_window_size(1 << 27)
    d.trace_enable()
    r = d.reset(frame)
    d.decode_blocks(r)
    out = d.collect()
    _, _, seqs = d.trace()
    assert d.window_size() == 1 << window_log
    assert len(seqs) == 0 or int(seqs[:, 3].max()) <= 1 << window_log
    assert out == data
    assert datagen.decompress(frame, len(data), window_log_max=27) == data
    return seqs


MIXED = planted(1400000, [(1000000, 1000, 299000), (700000, 400000, 50000), (1300000, 150000, 30000)], 1)


@pytest.mark.parametrize("lazy", [False, True], ids=["fastest", "lazy"])
@pytest.mark.parametrize("window_log", [18, 23])
def test_model_frames_decode_within_their_window(oracle, lazy, window_log):
    level = clazy.LAZY if lazy else cparse.FASTEST
    blocks = cldm.parse([MIXED], window_log, level=level)[0]
    frame = cparse.reference_frame(MIXED, blocks, level=level, window_log=window_log)
    wl = cparse.frame_window_log(len(MIXED), window_log)
    seqs = decode_checked(oracle, frame, MIXED, wl)
    offs = cldm.offsets(blocks)
    far = [o for o in offs if o > cldm.WINDOW]
    assert all(o <= 1 << window_log for o in offs)
    # the third repeat's source also lies inside the first one's copy, 151000 bytes back: the nearest earlier anchor wins
    if window_log == 23:
        assert set(far) == {999000, 300000, 151000}
        assert len(frame) < len(MIXED) - 350000
    else:
        assert set(far) == {151000}
    assert len(seqs) == len(offs)


def test_anchors_are_content_defined():
    data = planted(300000, [], 2)
    pos, keys = cldm.anchors(data)
    assert len(pos) > 300000 // 256
    for k in (1, 7, 1000):
        pre = bytes(np.random.default_rng(k).integers(0, 256, k, dtype=np.uint8).tobytes())
        p2, k2 = cldm.anchors(pre + data)
        edge = cldm.LDM_LEN - 1 + cldm.LDM_QUIET
        a = {(int(p) + k, int(x)) for p, x in zip(pos, keys) if p >= edge}
        b = {(int(p), int(x)) for p, x in zip(p2, k2) if p >= k + edge}
        assert a == b


@pytest.mark.parametrize("name", ["zeros"] + [f"period{p}" for p in range(1, 17)] + ["random", "text"])
def test_density_bound(name):
    n = 1 << 18
    if name == "zeros":
        data = bytes(n)
    elif name == "random":
        data = planted(n, [], 3)
    elif name == "text":
        data = bytes(datagen.gen_text(n, 4))
    else:
        p = int(name[6:])
        unit = planted(p, [], 100 + p)
        data = (unit * (n // p + 1))[:n]
    pos, _ = cldm.anchors(data)
    assert len(pos) <= -(-n // (cldm.LDM_QUIET + 1))
    assert len(pos) < 2 or int(np.diff(pos).min()) >= cldm.LDM_QUIET + 1


@pytest.mark.parametrize("window_log", [18, 23, 27])
def test_kept_matches(window_log):
    frames = [MIXED, planted(600000, [(400000, 100, 150000)], 5)]
    for f, blocks in zip(frames, cldm.forced(frames, window_log)):
        assert len(blocks) == -(-len(f) // BLOCK)
        for b, kept in enumerate(blocks):
            b0, n = b * BLOCK, min(BLOCK, len(f) - b * BLOCK)
            end = 0
            for s, ln, off in kept:
                assert 0 <= s and s + ln <= n and ln >= cldm.LDM_LEN and s >= end
                assert cldm.WINDOW < off <= 1 << window_log and b0 + s - off >= 0
                assert f[b0 + s:b0 + s + ln] == f[b0 + s - off:b0 + s - off + ln]
                end = s + ln


@pytest.mark.parametrize("off,window_log,taken", [(131072, 27, False), (131073, 27, True), (1 << 18, 18, True), ((1 << 18) + 1, 18, False),
                                                  (1 << 20, 20, True), ((1 << 20) + 1, 20, False)])
def test_offset_edges(off, window_log, taken):
    data = planted(off + 9000, [(off + 3000, 3000, 4000)], 6)
    offs = {o for blocks in cldm.forced([data], window_log) for kept in blocks for _, _, o in kept}
    assert offs == ({off} if taken else set())


def test_identical_frames_do_not_match_each_other():
    a = planted(300000, [], 7)
    kept = cldm.forced([a, a, a], 27)
    assert all(not k for blocks in kept for k in blocks)
    b = planted(400000, [(300000, 1000, 60000)], 8)
    kept = cldm.forced([a, b, a], 27)
    assert [len(k) for k in kept[1]] == [0, 0, 1, 0] and all(not k for k in kept[0] + kept[2])


def test_small_frames_are_the_regular_parse():
    f = planted(BLOCK, [(100000, 100, 20000)], 9)
    for level in (cparse.FASTEST, clazy.LAZY):
        assert cldm.parse([f], 27, level=level) == cparse.parse([f], level=level)


def test_window_descriptor_rule(tmp_path):
    exe = str(tmp_path / "frame_window_test")
    subprocess.check_call([seqcraft.NVCC, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe,
                           os.path.join(seqcraft.HERE, "host", "frame_window_test.cpp")])
    sizes = [0, 1, BLOCK - 1, BLOCK, BLOCK + 1, 1 << 18, (1 << 18) + 1, 5 << 20, 1 << 27, (1 << 27) + 1, 1 << 32]
    cases = [(n, w) for n in sizes for w in (17, 18, 20, 23, 27)]
    out = subprocess.run([exe] + [f"{n}:{w}" for n, w in cases], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    rows = out.stdout.split("\n")[:-1]
    assert len(rows) == len(cases)
    for (n, w), row in zip(cases, rows):
        hexhdr, wl, st, ws = row.split()
        want = min(w, max(17, (n - 1).bit_length() if n > 1 else 0))
        assert int(wl) == want == cparse.frame_window_log(n, w), (n, w)
        assert int(st) == 0 and int(ws) == 1 << want
        hdr = bytes.fromhex(hexhdr)
        assert hdr[5] == (want - 10) << 3
        assert hdr == cparse.frame_header(n, True, window_log=w)
        if n <= BLOCK:
            assert hdr[5] == 0x38
