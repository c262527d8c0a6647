"""CPU tests of the execution-kernel LOGIC (tests/emul_exec_cta.py models zstd-rs_b200/csrc/exec_cta.cuh bit by bit):
the oracle's per-block traces ({ll, ml, offset_value}, literals) are turned into what k_fse hands over -- prefix-form
records with symbolic offsets -- and executed by the model; the result must be the reference's output of that block."""
import numpy as np

from conftest import read_golden
import emul_exec_cta as E


def test_model_on_corpus_frames(oracle, manifest):
    """a handful of decodecorpus frames (multi-block, repeat offsets, RLE/raw literals, far matches)"""
    names = sorted(manifest["corpus"])
    picked = [n for n in names if manifest["corpus"][n]["size"] < 40000][:14] + ["z000003.zst"]   # z000003: 137 small blocks, far sources into row 0
    nb = ns = 0
    for n in picked:
        b, s = E.run_frame(oracle, read_golden("decodecorpus", n))
        nb += b; ns += s
    assert nb > 20 and ns > 2000


def test_model_on_synthetic(oracle):
    """libzstd level-3 frames: text-like (many short sequences), long overlapping runs, a 2-block chained frame"""
    import datagen as G
    rng = np.random.Generator(np.random.PCG64(5))
    words = [bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(300)]
    text = b" ".join(words[int(i)] for i in rng.integers(0, 300, 9000))[:48000]
    runs = b"".join(bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 700)) for _ in range(60)) + b"abcabcabc" * 500 + b"xy" * 3000
    chained = (text * 4)[:150000]   # > 128 KiB: two chained blocks, matches reach into the first block
    # a block that is nearly all literals (low-entropy bytes without matches): the literals do not fit beside the window
    lowent = bytes(rng.choice(np.arange(40, 56, dtype=np.uint8), 126000, p=np.arange(1, 17) / 136.0)) + text[:4000]
    for plain, mb in ((text, None), (runs, None), (chained, None), (lowent, None)):
        frame = G.compress(np.frombuffer(plain, dtype=np.uint8), level=3)
        nb, ns = E.run_frame(oracle, frame, mb)
        assert nb >= 1


def test_symbolic_history_matches_reference_rule():
    """sequence_execution.rs:125-133: of == 3, ll == 0, hist[0] == 0 -> 0 (saturating), through the symbolic form"""
    sym, h = E.symbolic_offsets([0], [3])
    assert E.sym_resolve(int(sym[0]), [0, 4, 8]) == 0
    assert E.sym_resolve(int(sym[0]), [1, 4, 8]) == 0
    assert E.sym_resolve(int(sym[0]), [7, 4, 8]) == 6
    # three decrements in a row stay saturating
    sym, h = E.symbolic_offsets([0, 0, 0], [3, 3, 3])
    assert [E.sym_resolve(int(v), [2, 9, 9]) for v in sym] == [1, 0, 0]
