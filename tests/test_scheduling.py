"""CPU tests of a submission's scheduling decisions (csrc/plan.cpp, through the host-only debug entries of the C ABI): which
execution kernel takes the multi-block frames, and the order in which k_fse takes the blocks.  No GPU involved."""
import numpy as np


def _w(nseq, comp):
    return int(nseq + comp // 16)


def test_routing_crossover_on_similar_frames(pkg):
    """1 MiB Silesia-mix-shaped frames (~70 k sequences, ~410 KB compressed): few frames -> one CTA each, thousands -> one warp each
    (the crossover of the cost model in csrc/plan.cpp lies between 1,024 and 2,048 frames on the 132 SMs of an H100)."""
    rng = np.random.Generator(np.random.PCG64(5))
    for n, expect_cta in ((8, True), (64, True), (512, True), (1024, True), (2048, False), (4096, False), (20000, False)):
        work = [_w(int(70000 * rng.uniform(0.1, 1.65)), int(410000 * rng.uniform(0.15, 2.3))) for _ in range(n)]
        cta = pkg.binding.route_frames(work, np.ones(n, dtype=np.uint8))
        assert len(cta) in (0, n), (n, len(cta))          # similar frames: never a split
        assert (len(cta) == n) == expect_cta, (n, len(cta))
        if len(cta):
            w = np.array(work)[cta]
            assert (np.diff(w.astype(np.int64)) <= 0).all()      # largest first: the ticket order of k_exec_cta
            assert sorted(cta.tolist()) == list(range(n))


def test_routing_keeps_ineligible_frames_on_the_warp_kernel(pkg):
    n = 300
    work = [_w(70000, 410000)] * n
    el = np.ones(n, dtype=np.uint8)
    el[::3] = 0                                        # dictionary / single-block / tiny frames
    cta = pkg.binding.route_frames(work, el)
    assert set(cta.tolist()) == set(np.nonzero(el)[0].tolist())
    assert len(pkg.binding.route_frames(work, np.zeros(n, dtype=np.uint8))) == 0
    assert len(pkg.binding.route_frames([], [])) == 0


def test_routing_few_large_frames_and_a_crowd(pkg):
    """A few long chained frames take CTAs whatever else is in the submission (a warp would need seconds for them); with a crowd of
    small multi-block frames beside them the model may split the list, but never leaves a long chain to a warp."""
    big = [_w(1_290_000, 5_900_000)] * 8                 # 16 MiB chained text frames
    cta = pkg.binding.route_frames(big, np.ones(8, dtype=np.uint8))
    assert sorted(cta.tolist()) == list(range(8))
    one = pkg.binding.route_frames([_w(82_000_000, 378_000_000)], [1])    # ONE chained 1 GiB frame
    assert one.tolist() == [0]
    crowd = big + [_w(6000, 40000)] * 6000
    cta = pkg.binding.route_frames(crowd, np.ones(len(crowd), dtype=np.uint8))
    assert set(range(8)) <= set(cta.tolist())


def test_fse_order_is_a_row_major_permutation(pkg):
    rng = np.random.Generator(np.random.PCG64(6))
    nframes = 200
    nblocks = rng.integers(1, 12, nframes).astype(np.uint32)
    first = np.concatenate([[0], np.cumsum(nblocks)[:-1]]).astype(np.uint32)
    total = int(nblocks.sum())
    nseq = rng.integers(0, 20000, total).astype(np.uint32)
    on_cta = (rng.random(nframes) < 0.2).astype(np.uint8)
    order = pkg.binding.fse_order(first, nblocks, on_cta, nseq)
    assert sorted(order.tolist()) == list(range(total))                   # a permutation of the blocks
    frame_of = np.repeat(np.arange(nframes), nblocks)
    row_of = np.concatenate([np.arange(n) for n in nblocks])
    warp_blocks = int(nblocks[on_cta == 0].sum())
    head, tail = order[:warp_blocks], order[warp_blocks:]
    assert (on_cta[frame_of[head]] == 0).all() and (on_cta[frame_of[tail]] == 1).all()     # k_exec_cta's frames last ...
    assert tail.tolist() == [b for b in range(total) if on_cta[frame_of[b]]]               # ... frame after frame
    rows = row_of[head]
    assert (np.diff(rows) >= 0).all()                                                       # row by row
    for r in range(int(rows.max()) + 1):
        seg = head[rows == r]
        assert len(seg) == int(((nblocks > r) & (on_cta == 0)).sum())                       # one block of every frame that has row r
        assert (np.diff(nseq[seg].astype(np.int64)) <= 0).all()                             # longest chains first inside the row


def test_fse_order_left_empty_when_it_would_not_matter_or_cannot_be_trusted(pkg):
    n = 50
    ones = np.ones(n, dtype=np.uint32)
    first = np.arange(n, dtype=np.uint32)
    assert len(pkg.binding.fse_order(first, ones, np.zeros(n, dtype=np.uint8), np.full(n, 7, dtype=np.uint32))) == 0     # single-block frames
    two = np.full(n, 2, dtype=np.uint32)
    first2 = (2 * np.arange(n)).astype(np.uint32)
    assert len(pkg.binding.fse_order(first2, two, np.ones(n, dtype=np.uint8), np.full(2 * n, 7, dtype=np.uint32))) == 0  # every frame on CTAs
    assert len(pkg.binding.fse_order(first2, two, np.zeros(n, dtype=np.uint8), np.full(2 * n + 3, 7, dtype=np.uint32))) == 0   # blocks outside any frame
    overlap = first2.copy(); overlap[1] = 1
    assert len(pkg.binding.fse_order(overlap, two, np.zeros(n, dtype=np.uint8), np.full(2 * n, 7, dtype=np.uint32))) == 0       # overlapping frames
    assert len(pkg.binding.fse_order(first2, two, np.zeros(n, dtype=np.uint8), np.full(2 * n, 7, dtype=np.uint32))) == 2 * n
