"""The compressor's frame header with a dictionary ID (no GPU needed): write_frame_header (zstd-rs_b200/csrc/encode.cuh), host-compiled,
against an independent Python writer, and read back with the decoder's parse_frame_header (zstd-rs_b200/csrc/framing.cuh)."""
import os
import shutil
import struct
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def py_frame_header(n, dict_id, checksum):
    """Single_Segment = 0, window descriptor 128 KiB, the dictionary ID in the smallest field that holds it (none for 0), then
    Frame_Content_Size in the smallest legal field (2 bytes hold 256..65791, stored minus 256)."""
    did = b"" if dict_id == 0 else struct.pack("<B", dict_id) if dict_id < 256 else struct.pack("<H", dict_id) if dict_id < 65536 else struct.pack("<I", dict_id)
    did_flag = {0: 0, 1: 1, 2: 2, 4: 3}[len(did)]
    if 256 <= n <= 65791:
        fcs, flag = struct.pack("<H", n - 256), 1
    elif n >> 32:
        fcs, flag = struct.pack("<Q", n), 3
    else:
        fcs, flag = struct.pack("<I", n), 2
    return struct.pack("<IBB", 0xFD2FB528, (flag << 6) | (4 if checksum else 0) | did_flag, 7 << 3) + did + fcs


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not available")
def test_frame_header_with_dictionary_id(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "frame_header_test")
    subprocess.check_call([nvcc, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe, os.path.join(HERE, "host", "frame_header_test.cpp")])
    ids = [0, 1, 255, 256, 65535, 65536, (1 << 32) - 1]
    sizes = [0, 255, 256, 65791, 65792, (1 << 32) - 1, 1 << 32]   # the 4-, 2- and 8-byte content size fields and their edges
    cases = [(n, i, c) for n in sizes for i in ids for c in (0, 1)]
    out = subprocess.run([exe] + [f"{n}:{i}:{c}" for n, i, c in cases], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    rows = out.stdout.split("\n")[:-1]
    assert len(rows) == len(cases)
    for (n, i, c), row in zip(cases, rows):
        hexhdr, size, status, has_id, dict_id, fcs, csum, wd, hsize = row.split()
        want = py_frame_header(n, i, c)
        assert bytes.fromhex(hexhdr) == want, (n, i, c)
        assert int(size) == int(hsize) == len(want), (n, i, c)
        assert (int(status), int(has_id), int(dict_id), int(fcs), int(csum), int(wd)) == (0, 1 if i else 0, i, n, c, 7 << 3), (n, i, c, row)
