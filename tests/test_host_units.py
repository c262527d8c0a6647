"""Host-compiled unit checks of device/host shared code (no GPU needed: nvcc compiles the __host__ __device__ helpers for the host)."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not available")
def test_description_bit_readers_match_bit_serial_reference(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "bit_readers_test")
    subprocess.check_call([nvcc, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe, os.path.join(HERE, "host", "bit_readers_test.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_bench_reference_arm_line(tmp_path):
    """`bench.py --impl reference` (the restated CPU path on the host cores) prints the contract's JSON line on a small workload."""
    import json
    import sys
    root = os.path.dirname(HERE)
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--frames", "64", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "decompressed_GBps" and line["unit"] == "GB/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"] == {"value": line["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


# ---- the header parsers shared by the host planner and k_walk (zstd-rs_b200/csrc/framing.cuh), host-compiled
STAGE_BLOCK_BODY, STAGE_LITERALS = 3, 4
HS_BEFORE_LITERALS = 1


@pytest.fixture(scope="module")
def framing(tmp_path_factory):
    """Runs tests/host/framing_test.cpp on a list of ("F" | "S", bytes) cases; returns one tuple of ints per case."""
    if shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("nvcc not available")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    d = tmp_path_factory.mktemp("framing")
    exe = str(d / "framing_test")
    subprocess.check_call([nvcc, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe, os.path.join(HERE, "host", "framing_test.cpp")])

    def run(cases):
        path = d / "cases.txt"
        path.write_text("".join(f"{kind} {data.hex()}\n" for kind, data in cases))
        out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        rows = [tuple(int(x) for x in r.split()) for r in out.stdout.splitlines()]
        assert len(rows) == len(cases)
        return rows
    return run


def _oracle_error(fn):
    from oracle import oracle as O
    try:
        fn()
        return 0, 0
    except O.OracleError as x:
        return x.code, x.stage


def test_frame_header_parse_matches_oracle_reset(framing, oracle):
    """Every descriptor byte with four choices of the field bytes, cut at every length up to one byte past the header, plus skippable
    and wrong magic numbers: the shared parser, read the way the frame decoder's reset reads, must give FrameDecoder.reset's error
    and take the same bytes from the source (all of the header and nothing past it)."""
    magic = bytes([0x28, 0xB5, 0x2F, 0xFD])
    tail = bytes([0x01, 0x02, 0x03])   # what follows the header: a block header
    srcs = []
    for desc in range(256):
        for fields in (bytes(13), b"\xff" * 13, bytes([desc]) + bytes(range(1, 13)), bytes([(desc * 37) & 0xFF]) + bytes(12)):
            single, flag = (desc >> 5) & 1, desc >> 6
            n = (1 - single) + [0, 1, 2, 4][desc & 3] + ([single, 2, 4, 8][flag])
            full = magic + bytes([desc]) + fields[:n] + tail
            srcs += [full[:k] for k in range(0, 5 + n + 2)]
    for m in list(range(0x184D2A4F, 0x184D2A61)) + [0xFD2FB527, 0xFD2FB529, 0x28B52FFD, 0]:
        full = m.to_bytes(4, "little") + bytes([7, 1, 0, 0, 0xAA])
        srcs += [full[:k] for k in range(0, len(full) + 1)]
    got = framing([("F", s) for s in srcs])
    dec = oracle.FrameDecoder()
    names = {v: k for k, v in oracle.error_names().items()}
    seen = set()
    for s, (e, taken) in zip(srcs, got):
        r = oracle._Reader(s)
        want = _oracle_error(lambda: dec.reset(r))[0]
        assert (e, taken) == (want, r.src.tell()), (s.hex(), e, taken, want, r.src.tell())
        seen.add(e)
    assert seen == {0} | {names["ZO_ERR_" + n] for n in (
        "MAGIC_NUMBER_READ", "BAD_MAGIC_NUMBER", "FRAME_DESCRIPTOR_READ", "WINDOW_DESCRIPTOR_READ", "DICTIONARY_ID_READ",
        "FRAME_CONTENT_SIZE_READ", "SKIP_FRAME", "WINDOW_TOO_BIG", "WINDOW_SIZE_TOO_BIG", "DICT_NOT_PROVIDED")}   # (no window descriptor is too small)


def _compressed_blocks(frames):
    """(content, (literals header fields), (sequences header fields)) of every Compressed block, located and parsed by tests/refwalk.py"""
    import numpy as np
    import refwalk
    bd = np.dtype([(k, "u8") for k in ("src_off", "content_size", "block_type", "last_block", "decompressed_size", "literals_type",
                                        "regenerated_size", "compressed_size", "num_streams", "num_sequences", "modes")])
    bf = np.dtype([(k, "u8") for k in ("out_off", "out_cap", "window_size", "first_block", "num_blocks")])
    comp, blocks, _ = refwalk.walk(frames, [0] * len(frames), [0] * len(frames), (bd, bf))
    comp = comp.tobytes()
    for b in blocks:
        if b["block_type"] == 2:
            c = comp[int(b["src_off"]):int(b["src_off"] + b["content_size"])]
            lt, regen, csize, streams, n, payload = refwalk.literals_header(c)
            s = c[n + payload:]
            nseq, modes = refwalk.sequences_header(s)
            hdr = 1 if s[0] == 0 else 2 if s[0] < 128 or (s[0] < 255 and nseq == 0) else 3 if s[0] < 255 else 4
            yield c, (lt, streams, regen, csize, n), (nseq, modes if nseq else None, n + payload + hdr)


def test_section_headers_of_golden_frames_match_refwalk(framing, manifest):
    """Every Compressed block of the golden corpus and the dictionary frames: the shared section parser's fields equal refwalk's."""
    from conftest import read_golden
    frames = [read_golden("decodecorpus", n) for n in sorted(manifest["corpus"])]
    frames += [read_golden("dict_tests", "files", n) for n in sorted(manifest["dict"])]
    blocks = list(_compressed_blocks(frames))
    assert len(blocks) > 1000
    got = framing([("S", c) for c, _, _ in blocks])
    for (c, lit, seq), (status, lt, streams, regen, csize, lit_off, nseq, modes, seq_off) in zip(blocks, got):
        assert status == 0 and (lt, streams, regen, csize, lit_off) == lit, (c[:8].hex(), lit)
        assert (nseq, modes if nseq else None, seq_off) == seq, (c[:8].hex(), seq)


def _crafted_contents():
    """Compressed block contents of 0..8 bytes: every literals header first byte, two fillings of the rest of the literals header,
    then a sequences header prefix where the literals section says it starts (refwalk), cut at every length."""
    import random
    import refwalk
    rng = random.Random(11)
    prefixes = [b"", b"\x00", b"\x00\x00", b"\x05", b"\x05\x00", b"\x7f\xfc", b"\x80\x00", b"\x80\x00\x00", b"\x80\x03", b"\x80\x03\x00",
                b"\xfe\xff\x54", b"\xff", b"\xff\x01", b"\xff\x01\x02", b"\xff\x01\x02\x00", b"\xff\x01\x02\x00\x00"]
    out = {b""}
    for b0 in range(256):
        for rest in (bytes(4), bytes(rng.randrange(256) for _ in range(4))):
            c = bytes([b0]) + rest
            _, _, _, _, n, payload = refwalk.literals_header(c)
            head = c[:n] + bytes(rng.randrange(256) for _ in range(min(payload, 8)))
            for s in prefixes:
                full = head + s + b"\x00\x01"
                out.update(full[:k] for k in range(1, 9))
    return sorted(out)


def test_section_headers_of_crafted_blocks_match_oracle(framing, oracle):
    """One-block frames around the crafted contents: where the shared parser reports an error before the literals stage, the oracle
    reports the same code and stage; an error after it is the oracle's too, unless the literals stage failed first (the order
    block_first_error reports them in); where the parser reports none, any error of the oracle comes from a later stage, and from
    the literals stage when there are no sequences."""
    contents = _crafted_contents()
    assert len(contents) > 10000
    got = framing([("S", c) for c in contents])
    dec = oracle.FrameDecoder()
    seen = {"before": 0, "after": 0, "after_lit_first": 0, "none": 0}
    for c, row in zip(contents, got):
        status = row[0]
        frame = bytes([0x28, 0xB5, 0x2F, 0xFD, 0x00, 0x00]) + ((len(c) << 3) | (2 << 1) | 1).to_bytes(3, "little") + c

        def run():
            r = dec.reset(frame)
            dec.decode_blocks(r)
        code, stage = _oracle_error(run)
        mine = (status & 0xFFFF, (status >> 16) & 0xFF)
        if status and status >> 24 == HS_BEFORE_LITERALS:
            assert (code, stage) == mine, (c.hex(), mine, code, stage)
            seen["before"] += 1
        elif status:
            assert (code, stage) == mine or stage == STAGE_LITERALS, (c.hex(), mine, code, stage)
            seen["after" if (code, stage) == mine else "after_lit_first"] += 1
        else:   # (with no sequences, nothing runs after the literals stage)
            assert code == 0 or (stage == STAGE_LITERALS if row[6] == 0 else stage >= STAGE_LITERALS), (c.hex(), code, stage)
            seen["none"] += 1
    assert min(seen.values()) > 100, seen
