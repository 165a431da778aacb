"""The survivor model without a GPU (tests/_survivor_model.py; tests/test_survivors.py is the GPU half).

- The batch packing restated in the model has the engine's constants, and at every block size and tail the GPU file
  runs, the edge-crossing mask really straddles every batch edge (and every lane edge with three lanes), the buffers
  span at least three batches, and a batch closes at the limit the case is there for.
- The canary differs from the source in every byte.
- check_image catches an engine that writes one block past the end of each survivor run, and one that writes a single
  skipped block, and names the first wrong block; it passes the correct image."""
import re
from pathlib import Path

import numpy as np
import pytest

import _survivor_model as sm
from _survivor_model import MiB

CSRC = Path(__file__).resolve().parent.parent / "gpu-docker-api_b200" / "csrc"
SLOT = sm.DEFAULT_SLOT
BBS = [4096, 12288, 65536, MiB + 4096, 4 * MiB, SLOT]
BB_IDS = ["4K", "12K", "64K", "1M+4K", "4M", "slot"]


def _span_blocks(bb, slot, lanes=1):
    cap = sm.batch_capacity(bb, slot)
    return lanes * (2 * cap + max(1, cap // 4))


def _const(path, pattern):
    m = re.search(pattern, (CSRC / path).read_text())
    assert m, (path, pattern)
    return int(m.group(1))


def test_model_constants_are_the_engines():
    assert _const("vmig_engine.cu", r"kMaxBatchBlocks\s*=\s*(\d+)\s*;") == sm.MAX_BATCH_BLOCKS
    assert _const("vmig_kernels.cuh", r"kBlockAlign\s*=\s*(\d+)\s*;") == sm.BLOCK_ALIGN
    assert _const("vmig_engine.cu", r'env_long\("VMIG_SLOT_MB",\s*(\d+)\)') << 20 == sm.DEFAULT_SLOT
    # the batch planner's rule, as run_lane states it
    src = (CSRC / "vmig_engine.cu").read_text()
    assert "align_up(std::max<uint32_t>(blocks[i].len, 1), blk_align)" in src
    assert "if (used + need > slot_bytes) break;" in src


# the block sizes of tests/test_survivors.py at the default slot, and those of its child run at the 4 MiB minimum
EDGE_CASES = [(bb, SLOT) for bb in BBS] + [(4 * MiB, 4 * MiB), (4096, 4 * MiB)]


@pytest.mark.parametrize("bb,slot", EDGE_CASES, ids=[f"{i}-slot{s >> 20}M" for i, (_, s) in zip(BB_IDS + ["4M", "4K"], EDGE_CASES)])
def test_edge_masks_straddle_every_batch_edge(bb, slot):
    k = _span_blocks(bb, slot)
    for tail in (0, 1, 31, bb - 1):
        n = k * bb + tail
        lens = sm.block_lens(n, bb)
        batches = sm.pack_batches(lens, slot)
        assert len(batches) >= 3, (bb, tail, batches[:4])
        assert batches[0][0] == 0 and batches[-1][1] == lens.size
        assert all(a[1] == b[0] for a, b in zip(batches, batches[1:]))
        want = np.arange(lens.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        prior = dict((name, p) for name, p, _ in sm.families(want, lens, bb, slot, seed=0))["batch_edges"]
        m = prior != want
        for b0, _ in batches[1:]:
            assert m[b0 - 1] and m[b0], (bb, tail, b0)


def test_batches_close_at_the_limit_each_block_size_is_there_for():
    def first(bb, slot):
        lens = sm.block_lens(_span_blocks(bb, slot) * bb, bb)
        b0, b1 = sm.pack_batches(lens, slot)[0]
        return b1 - b0, (b1 - b0) * sm.align_up(bb, sm.BLOCK_ALIGN)
    assert first(4096, SLOT) == (sm.MAX_BATCH_BLOCKS, 16 * MiB)            # the block cap, half the slot used
    assert first(12288, SLOT)[0] == SLOT // 12288 < sm.MAX_BATCH_BLOCKS     # the slot fills first
    assert first(MiB + 4096, SLOT)[0] == 31                                  # 31 blocks; a 32nd overflows the slot
    assert first(SLOT, SLOT)[0] == 1
    assert first(4 * MiB, 4 * MiB)[0] == 1                                   # the minimum slot: one block per launch
    assert first(4096, 4 * MiB) == (1024, 4 * MiB)                           # the slot fills before the block cap
    # a short tail block takes 512 bytes of a slot, a 1-byte block too, and a 0-byte block still one aligned unit
    assert sm.pack_batches(np.array([SLOT - 512, 1, 0], np.uint32), SLOT) == [(0, 2), (2, 3)]


def test_three_lanes_deal_blocks_round_robin_or_split_ranges():
    lens = sm.block_lens(10 * 4096 + 31, 4096)
    assert [s.tolist() for s in sm.lane_shares(lens, 3)] == [[0, 3, 6, 9], [1, 4, 7, 10], [2, 5, 8]]
    lens = sm.block_lens(4 * 4 * MiB + 31, 4 * MiB)         # 5 blocks: fewer than two per lane; the 31-byte one weighs 4096
    assert [s.tolist() for s in sm.lane_shares(lens, 3)] == [[0, 1], [2], [3, 4]]
    # every lane of the 3-lane case packs at least three batches, and the mask holds both sides of every lane's
    # batch edges and each lane's first and last block
    lens = sm.block_lens(_span_blocks(4096, SLOT, 3) * 4096 + 31, 4096)
    shares = sm.lane_shares(lens, 3)
    assert all(len(sm.pack_batches(lens[s], SLOT)) >= 3 for s in shares)
    assert sm.launches(lens, SLOT, 3) == sum(len(sm.pack_batches(lens[s], SLOT)) for s in shares)
    want = np.arange(lens.size, dtype=np.uint64) + np.uint64(1)
    prior = dict((name, p) for name, p, _ in sm.families(want, lens, 4096, SLOT, seed=0, lanes=3))["batch_edges"]
    m = prior != want
    pairs = sm.edge_pairs(lens, SLOT, 3)
    assert len(pairs) >= 6 and all(m[a] and m[b] for a, b in pairs)
    assert all(m[a] and m[b] for a, b in sm.lane_ends(lens, 3))


def test_masks_are_what_their_names_say():
    bb, n = 4096, 300 * 4096 + 1
    lens = sm.block_lens(n, bb)
    want = np.arange(lens.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(7)
    got = {name: sm.survivors(want, p, v) for name, p, v in sm.families(want, lens, bb, SLOT, seed=0)}
    nb = lens.size
    assert got["no_table"].all() and not got["none"].any() and got["all"].all()
    assert got["first_only"].tolist() == [True] + [False] * (nb - 1)
    assert got["last_only"].tolist() == [False] * (nb - 1) + [True]
    assert sm.mask_runs(got["run_65"]) == [(nb // 3, nb // 3 + 65)]
    long_run = MiB // bb + 1                                        # 257 blocks: the run is moved back to fit
    assert sm.mask_runs(got["run_1MiB_plus_1"]) == [(nb - long_run, nb)]
    assert 0 < got["random_1"].sum() < nb // 20 and 0 < (~got["random_99"]).sum() < nb // 20
    v0 = got["valid0_prior_equal"]
    assert v0[3] and v0[10] and v0[-1] and not v0[4] and v0.sum() == len(range(3, nb, 7)) + 1
    for name, bit in (("bit0", 0), ("bit63", 63)):
        p = dict((k, p) for k, p, _ in sm.families(want, lens, bb, SLOT, seed=0))[name]
        d = p ^ want
        assert set(d[d != 0].tolist()) == {1 << bit} and (got[name] == (d != 0)).all()


# ------------------------------------------------------------------------------------------ the image check
def _case(bb, tail, k=40, seed=0x77):
    from oracle import oracle
    n = k * bb + tail
    src = oracle.splitmix_bytes(seed, n + 4096).copy()
    return n, src, sm.canary_for(src, seed + 1)


def test_canary_differs_from_the_source_in_every_byte():
    _, src, canary = _case(4096, 31)
    assert (canary != src).all()
    w = src.size // 8 * 8
    assert (canary[:w].view(np.uint64) != src[:w].view(np.uint64)).all()


def _engine(src, canary, write, bb, n, bug=None):
    """The dst image a (possibly wrong) engine leaves."""
    img = canary.copy()
    sm.paint(img, src, write, bb, n)
    wrong = np.zeros_like(write)
    if bug == "past_run_end":                          # one block too many behind each run of survivors
        for _a, b in sm.mask_runs(write):
            if b < write.size:
                wrong[b] = True
    elif bug == "one_skipped":                          # one skipped block written
        wrong[np.flatnonzero(~write)[len(np.flatnonzero(~write)) // 2]] = True
    sm.paint(img, src, wrong, bb, n)
    return img, wrong


@pytest.mark.parametrize("bb", [4096, 65536])
@pytest.mark.parametrize("tail", [0, 1, 31])
@pytest.mark.parametrize("mask", ["alternating", "run_65", "random_50", "first_only", "valid0_prior_equal"])
def test_image_check_catches_wrong_engines(bb, tail, mask):
    n, src, canary = _case(bb, tail, k=200)
    lens = sm.block_lens(n, bb)
    want = np.arange(lens.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    p, v = {name: (p, v) for name, p, v in sm.families(want, lens, bb, SLOT, seed=5)}[mask]
    write = sm.survivors(want, p, v)
    good, _ = _engine(src, canary, write, bb, n)
    sm.check_image(good, src, canary, write, bb, n, mask)
    scratch = canary.copy()
    sm.check_image(good, src, canary, write, bb, n, mask, scratch)
    assert np.array_equal(scratch, canary)                          # used and given back
    for bug in ("past_run_end", "one_skipped"):
        img, wrong = _engine(src, canary, write, bb, n, bug)
        assert wrong.any(), (mask, bug)
        first = int(np.flatnonzero(wrong)[0])
        with pytest.raises(AssertionError, match=rf"block {first} \(skipped\) at byte 0 "):
            sm.check_image(img, src, canary, write, bb, n, mask, scratch)
        assert np.array_equal(scratch, canary)


def test_image_check_names_bytes_past_the_end_and_a_short_survivor():
    bb, tail = 4096, 31
    n, src, canary = _case(bb, tail)
    lens = sm.block_lens(n, bb)
    write = np.zeros(lens.size, bool)
    write[-1] = True
    img, _ = _engine(src, canary, write, bb, n)
    img[n + 5] ^= 1                                                 # a write of the aligned length, not the tail's
    with pytest.raises(AssertionError, match=rf"byte 5 past the end of the {n}-byte buffer"):
        sm.check_image(img, src, canary, write, bb, n, "tail")
    img, _ = _engine(src, canary, write, bb, n)
    img[n - 1] = canary[n - 1]                                      # the survivor's last byte not copied
    with pytest.raises(AssertionError, match=rf"block {lens.size - 1} \(written\) at byte {tail - 1} "):
        sm.check_image(img, src, canary, write, bb, n, "tail")
