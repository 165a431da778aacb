"""A plain numpy model of what a diff pass over a buffer must leave behind (vmig_migrate_buffer with a prior table).

K1 flags block b changed unless prior_valid[b] and prior[b] equals its hash; the engine D2H-copies and writes only the
changed blocks (the survivors), and include/vmig.h promises that "dst regions of skipped blocks are left untouched".
The tests fill dst with a canary that differs from src in every byte, so the image a call must leave is src over the
survivors and the canary everywhere else, up to and past the end of the buffer.

The engine's batch packing (run_lane in csrc/vmig_engine.cu) and the lane split of a buffer (run_blocks in
csrc/vmig_api.cu) are restated here, so that the masks that must straddle a batch or lane edge are computed from the
rule itself, and so that a test can hold the engine's kernel-launch count to the number of batches the rule makes."""
import numpy as np

from oracle import oracle

MiB = 1 << 20
MAX_BATCH_BLOCKS = 4096          # kMaxBatchBlocks: a batch closes at this many blocks ...
BLOCK_ALIGN = 512                # ... or when the next block, at align_up(max(len, 1), kBlockAlign), overflows the slot
DEFAULT_SLOT = 32 * MiB          # VMIG_SLOT_MB's default
LANE_MIN_BYTES = 4096            # the lane split weighs a block at max(len, 4096)


def align_up(v, a):
    return (v + a - 1) // a * a


def block_lens(n: int, bb: int) -> np.ndarray:
    nb = -(-n // bb)
    lens = np.full(nb, bb, np.uint32)
    if nb and n % bb:
        lens[-1] = n % bb
    return lens


def batch_capacity(bb: int, slot: int) -> int:
    """Full blocks of bb bytes in one batch."""
    return min(MAX_BATCH_BLOCKS, slot // align_up(bb, BLOCK_ALIGN))


def pack_batches(lens, slot: int):
    """[(b0, b1)] over positions of `lens`, in order, as run_lane packs one lane's block list."""
    out, i, n = [], 0, len(lens)
    while i < n:
        b0, used = i, 0
        while i < n and i - b0 < MAX_BATCH_BLOCKS:
            need = align_up(max(int(lens[i]), 1), BLOCK_ALIGN)
            assert need <= slot, (need, slot)
            if used + need > slot:
                break
            used += need
            i += 1
        out.append((b0, i))
    return out


def lane_shares(lens, lanes: int):
    """Table indices of each lane's blocks, in lane order.  A buffer has one write key per block, so with at least two
    blocks per lane the keys are dealt longest-first (ties by index) to the least-loaded lane (lowest index on ties):
    equal blocks go round-robin.  With fewer, the list is cut into contiguous ranges of about equal weight."""
    nb = len(lens)
    lanes = min(lanes, nb)
    if lanes <= 1:
        return [np.arange(nb)]
    w = np.maximum(np.asarray(lens, np.uint64), LANE_MIN_BYTES)
    lane_of = np.empty(nb, np.int64)
    if nb >= 2 * lanes:
        load = [0] * lanes
        for b in np.lexsort((np.arange(nb), -w.astype(np.int64))):
            best = min(range(lanes), key=lambda x: (load[x], x))
            load[best] += int(w[b])
            lane_of[b] = best
    else:
        total, acc, lane = int(w.sum()), 0, 0
        for b in range(nb):
            lane_of[b] = lane
            acc += int(w[b])
            if lane + 1 < lanes and acc >= total * (lane + 1) // lanes:
                lane += 1
    return [np.flatnonzero(lane_of == x) for x in range(lanes)]


def launches(lens, slot: int, lanes: int = 1) -> int:
    """K1 launches of a call: one per batch of every lane."""
    return sum(len(pack_batches(lens[s], slot)) for s in lane_shares(lens, lanes))


def edge_pairs(lens, slot: int, lanes: int = 1):
    """(last block of a batch, first block of the next batch of the same lane), as table indices."""
    out = []
    for s in lane_shares(lens, lanes):
        out += [(int(s[b0 - 1]), int(s[b0])) for b0, _ in pack_batches(lens[s], slot)[1:]]
    return out


def lane_ends(lens, lanes: int):
    """(first, last) table index of every lane's share."""
    return [(int(s[0]), int(s[-1])) for s in lane_shares(lens, lanes)]


def survivors(want, prior, valid) -> np.ndarray:
    """The blocks a diff pass must write: all of them without a prior table."""
    if prior is None:
        return np.ones(want.size, bool)
    return ~(np.asarray(valid).astype(bool) & (np.asarray(prior) == want))


def families(want, lens, bb: int, slot, seed: int, lanes: int = 1):
    """(name, prior, valid) over the true hashes `want` of blocks of bb bytes; prior None means no prior table.
    slot None leaves out the mask built from the batch and lane edges (a resident batch is one launch)."""
    nb = want.size
    i = np.arange(nb)
    one = np.ones(nb, np.uint8)

    def differ(mask, bit=0):
        p = want.copy()
        p[mask] ^= np.uint64(1 << bit)
        return p

    def run(start, length):
        start = max(0, min(start, nb - length))
        return (i >= start) & (i < start + length)

    yield "no_table", None, None
    yield "none", want, one
    yield "all", differ(i >= 0), one
    yield "alternating", differ(i % 2 == 1), one
    yield "first_only", differ(i == 0), one
    yield "last_only", differ(i == nb - 1), one
    yield "run_65", differ(run(nb // 3, 65)), one                                  # more than one 64-block writer task
    yield "run_1MiB_plus_1", differ(run(nb // 2, -(-MiB // bb) + 1)), one         # more than one 1 MiB writer task
    if slot is not None:
        m = np.zeros(nb, bool)
        for a, b in edge_pairs(lens, slot, lanes):
            m[max(a - 1, 0):a + 1] = True
            m[b:b + 2] = True
        for a, b in lane_ends(lens, lanes) if lanes > 1 else []:
            m[a] = m[b] = True
        yield "batch_edges", differ(m), one
    rng = np.random.default_rng(seed)
    for pct in (1, 50, 99):
        yield f"random_{pct}", differ(rng.random(nb) < pct / 100), one
    v = one.copy()
    v[(i % 7 == 3) | (i == nb - 1)] = 0
    yield "valid0_prior_equal", want, v
    yield "bit0", differ(i % 5 == 1, 0), one
    yield "bit63", differ(i % 5 == 2, 63), one


def canary_for(src: np.ndarray, seed: int) -> np.ndarray:
    """SplitMix64 stream `seed`, with every byte that happens to equal src's flipped: it differs from src in every
    byte, so a stray write of source bytes shows at its first byte."""
    c = oracle.splitmix_bytes(seed, src.size).copy()
    c[c == src] ^= 0x5A
    return c


def mask_runs(mask):
    """[(b0, b1)] of the maximal runs of True in mask."""
    m = np.concatenate(([False], np.asarray(mask, bool), [False]))
    d = np.flatnonzero(m[1:] != m[:-1])
    return list(zip(d[0::2].tolist(), d[1::2].tolist()))


def paint(target, source, mask, bb: int, n: int):
    """target := source over the bytes of the blocks in mask (the last block ends at n)."""
    for a, b in mask_runs(mask):
        target[a * bb:min(b * bb, n)] = source[a * bb:min(b * bb, n)]


def check_image(dst, src, canary, written, bb: int, n: int, what: str, scratch=None):
    """dst (canary-sized: the buffer and what lies past its end) must hold src over the written blocks and the canary
    everywhere else.  scratch, if given, is a copy of the canary that is used and restored instead of a new copy."""
    exp = canary.copy() if scratch is None else scratch
    paint(exp, src, written, bb, n)
    try:
        if np.array_equal(*(x.view(np.uint64) if x.size % 8 == 0 else x for x in (dst, exp))):      # 8 bytes a step
            return
        bad = np.flatnonzero(dst != exp)
        o = int(bad[0])
        if o >= n:
            where = f"byte {o - n} past the end of the {n}-byte buffer"
        else:
            b = o // bb
            where = f"block {b} ({'written' if written[b] else 'skipped'}) at byte {o - b * bb}"
        wrong = np.unique(np.minimum(bad // bb, written.size))
        raise AssertionError(f"{what}: {where} (offset {o}) holds {int(dst[o]):#04x}, want {int(exp[o]):#04x}; "
                             f"{wrong.size} wrong blocks, the first {wrong[:8].tolist()}")
    finally:
        if scratch is not None:
            paint(exp, canary, written, bb, n)
