"""CPU checks of the dictionary trainer's NumPy model (tests/dicttrain.py): the epoch rule, the rules for short inputs and small
dictionaries, sample boundaries, and the shape of a trained dictionary.  The GPU trainer is pinned to this model byte for byte
in test_gpu_dict_train.py."""
import numpy as np

import dicttrain as M


def compute_epoch_info(segment_size, max_dict_size, num_kmers):
    """ruzstd's compute_epoch_info (dictionary/cover.rs:117-132), line for line."""
    min_epoch_size = 10_000
    num_epochs = max(1, max_dict_size // segment_size)
    epoch_size = num_kmers // num_epochs
    if epoch_size >= min_epoch_size:
        assert epoch_size * num_epochs <= num_kmers
        return num_epochs, epoch_size
    epoch_size = min(min_epoch_size, num_kmers)
    num_epochs = num_kmers // epoch_size
    return num_epochs, epoch_size


def test_epoch_rule_matches_compute_epoch_info():
    branches = set()
    for n in (16, 17, 2047, 2048, 2049, 9999, 10000, 10001, 20000, 123457, 7 << 20, 345_000_000):
        for seg in (16, 256, 2048, 65536):
            for dict_size in (1, 100, 2047, 2048, 112640, 1 << 20, 10 * n):
                L = min(seg, n)
                E, es = compute_epoch_info(L, dict_size, n)
                assert M.epoch_info(n, dict_size, seg) == (E, es, L)
                branches.add(n // max(1, dict_size // L) >= 10_000)
                ep = M.epochs(n, dict_size, seg)
                assert len(ep) == E and ep[0][0] == 0 and ep[-1][1] == n
                assert all(a[1] == b[0] for a, b in zip(ep, ep[1:]))
                assert all(le == min(L, e1 - e0) and le >= 16 for e0, e1, le in ep)
    assert branches == {True, False}


def test_short_input_is_its_own_dictionary():
    for n in range(16):
        data = bytes(range(n))
        assert M.train(data, 100) == (data, [])
        assert M.train(data, 0) == (data, [])


def test_empty_dictionary():
    data = np.random.default_rng(1).integers(0, 256, 5000, dtype=np.uint8).tobytes()
    assert M.train(data, 0) == (b"", [])


def test_small_dictionary_keeps_the_tail():
    data = np.random.default_rng(2).integers(0, 40, 20000, dtype=np.uint8).tobytes()
    full, segs = M.train(data, 2048)
    assert len(segs) == 1 and len(full) == 2048
    for k in (1, 100, 2047):
        small, segs_k = M.train(data, k)
        assert small == full[-k:] and segs_k == segs


def test_kmer_across_a_sample_boundary_is_not_counted():
    rng = np.random.default_rng(3)
    P = b"0123456789abcdef"
    parts = []
    for _ in range(50):
        parts += [rng.integers(0, 256, 100, dtype=np.uint8).tobytes() + P[:8], P[8:] + rng.integers(0, 256, 60, dtype=np.uint8).tobytes()]
    data = b"".join(parts)
    sizes = [len(p) for p in parts]
    hp = M.slots(P)[0]
    one = M.slots(data)
    assert (one == hp).sum() == 50                   # one sample: the k-mer is there 50 times
    cut = M.slots(data, sizes)
    assert (cut == hp).sum() == 0                    # cut into samples: never
    end = 0
    for s in sizes:
        end += s
        assert (cut[end - 15:end] == M.NO_SLOT).all() and cut[end - 16] != M.NO_SLOT
    assert M.slots(b"x" * 15, [15]).tolist() == [M.NO_SLOT] * 15


def test_planted_phrase_once_and_best_last():
    rng = np.random.default_rng(4)
    data = bytearray(rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes())
    phrase = rng.integers(0, 256, 600, dtype=np.uint8).tobytes()
    for e in range(4):                               # 4 epochs of 25,000 bytes: 10 copies in each
        for j in range(10):
            at = e * 25_000 + 1000 + j * 2300
            data[at:at + 600] = phrase
    data = bytes(data)
    d, segs = M.train(data, 8192)
    assert len(segs) == 4 and len(d) == 8192
    assert d.count(phrase) == 1
    scores = [s[3] for s in sorted(segs, key=lambda t: (t[3], t[0]))]
    best = max(segs, key=lambda t: (t[3], -t[0]))
    assert d[-best[2]:] == data[best[1]:best[1] + best[2]] and scores[-1] == best[3]
    assert phrase in d[-2048:]
    assert best[3] > 2 * sorted(s[3] for s in segs)[-2]   # the later epochs got no credit for the phrase


def test_binding_buffers_hold_what_the_trainer_writes():
    """create_raw_dict sizes its buffers with binding.raw_dict_bounds; they must hold the exact need of the epoch rule."""
    import _pkg
    bounds = _pkg.load().binding.raw_dict_bounds
    for n in list(range(0, 40)) + [2047, 2048, 2049, 9999, 10000, 10001, 19999, 20000, 20001, 123457, 7 << 20, (1 << 32) - 1]:
        for seg in (16, 256, 2048, 65536):
            for dict_size in (0, 1, 100, 2048, 112640, 1 << 20, 10 * n + 1):
                cap, nseg = bounds(n, dict_size)
                if n < 16:
                    assert cap >= n
                    continue
                ep = M.epochs(n, dict_size, seg) if dict_size else []
                assert cap >= min(dict_size, sum(le for _, _, le in ep)) and nseg >= len(ep)
