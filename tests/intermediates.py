"""The decoder's intermediate results against the oracle's trace, block by block: what k_huf and k_fse left for one frame of a
prepared submission (Batch.debug_literals / debug_sequences / debug_block_flags)."""
import numpy as np


def check_intermediates(batch, blk, blocks, lits, seqs, label, hist=(1, 4, 8), exact=None, flags_exact=True):
    """Per block of one frame, from submission block index `blk` on: the literals k_huf decoded (debug_literals) and the
    sequences k_fse decoded (debug_sequences) against the oracle's trace `blocks, lits, seqs`; `hist` is the repeat-offset
    history at the frame's start.  With `exact` (exact_path_blocks), a block's raw-offset flag (debug_block_flags & 1) must be
    set exactly on the exact-path blocks -- or, when not `flags_exact`, only on them: k_exec_cta resolves a block's raw offsets
    in place and clears the flag.  Returns (next block index, literal sections checked, sequences checked)."""
    hist = list(hist)
    nlit = nseq = 0
    for k, tb in enumerate(blocks):
        if tb["block_type"] == 2:
            if tb["literals_type"] >= 2:
                got_l = batch.debug_literals(blk)
                assert got_l == lits[tb["lit_offset"]:tb["lit_offset"] + tb["regenerated_size"]], (label, blk)
                nlit += 1
            raw = batch.debug_block_flags(blk) & 1
            if exact is not None:
                assert (raw == exact[k]) if flags_exact else (not raw or exact[k]), (label, k, raw, exact[k])
            if tb["num_sequences"]:
                got_s = batch.debug_sequences(blk)
                exp = seqs[tb["seq_offset"]:tb["seq_offset"] + tb["num_sequences"]]
                assert np.array_equal(got_s[:, :2], exp[:, :2]), (label, blk)
                # offsets: raw offset_values when the block went through k_fse's exact path, otherwise already through
                # do_offset_history (oracle column 3), symbolic where they depend on the history at the block's start
                if raw:
                    assert np.array_equal(got_s[:, 2], exp[:, 2]), (label, blk)
                else:
                    sym = got_s[:, 2].astype(np.int64)
                    tag, dec = sym >> 30, sym & ((1 << 30) - 1)
                    h = np.array([0] + hist, dtype=np.int64)[tag]
                    actual = np.where(tag == 0, sym, np.maximum(h - dec, 0))
                    assert np.array_equal(actual, exp[:, 3].astype(np.int64)), (label, blk)
                nseq += len(exp)
                hist = list(tb["offset_hist_after"])
        blk += 1
    return blk, nlit, nseq
