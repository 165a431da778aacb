"""Diff-pass survivor tests (-m gpu): a buffer diff pass writes exactly the blocks K1 finds changed, and nothing else.

include/vmig.h promises that vmig_migrate_buffer leaves the dst regions of skipped blocks untouched.  Here dst starts as
a canary that differs from src in every byte, the prior table is built from the oracle's hashes and a mask, and after
each call dst must hold src over the survivors and the canary everywhere else, past the buffer's end included
(tests/_survivor_model.py); the hashes, the skip count, the D2H and written bytes and the K1 launch count must be what
the mask and the engine's batch packing imply.  That runs over the four memory configurations (the engine DMAs a
page-locked source or destination directly, a pageable one through the staging rings and the reader / writer
threads), block sizes on both sides of the batch limits, tail blocks of 0, 1, 31 and bb - 1 bytes, three lanes, one
staging slot, VMIG_F_HASH_ONLY and the minimum staging slot.  A resident batch checks K2's survivor list against the
same model.

Every expected value comes from the oracle's XXH64 and plain numpy, never from a second run of the engine."""
import functools
import os

import numpy as np
import pytest

from oracle import oracle
from _survivor_model import (DEFAULT_SLOT, MiB, batch_capacity, block_lens, canary_for, check_image, families,
                             launches, paint, survivors)
from test_geometry import _child_vm, _run_child

pytestmark = pytest.mark.gpu
SLOT = min(max(int(os.environ.get("VMIG_SLOT_MB", str(DEFAULT_SLOT >> 20))), 4), 1024) << 20
BBS = [4096, 12288, 65536, MiB + 4096, 4 * MiB, SLOT]
BB_IDS = ["4K", "12K", "64K", "1M+4K", "4M", "slot"]
MEMS = ["pageable-pageable", "pinned-pinned", "pinned-pageable", "pageable-pinned"]
GUARD = 4096                     # bytes past the buffer's end that must keep the canary
# the masks that also run at the 1- and 31-byte tails (every mask runs at tails 0 and bb - 1)
SHORT_TAIL_MASKS = {"no_table", "all", "last_only", "batch_edges", "random_50", "valid0_prior_equal"}


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def span_blocks(bb, slot, lanes=1):
    """Full blocks of a buffer whose every lane packs at least three batches."""
    cap = batch_capacity(bb, slot)
    return lanes * (2 * cap + max(1, cap // 4))


class Buffers:
    """src and dst of `size` bytes each, pinned (vm.PinnedBuffer) or pageable as `mem` says; src holds SplitMix64
    stream `seed`, dst and `canary` the canary, `scratch` a spare copy of it for check_image."""

    def __init__(self, vm, mem, size, seed):
        size = -(-size // 8) * 8
        self._pinned = []
        self.src, self.dst = (self._alloc(vm, kind, size) for kind in mem.split("-"))
        data = oracle.splitmix_bytes(seed, size)
        self.src[:] = data
        self.canary = canary_for(data, seed ^ 0xCA4A)
        self.dst[:] = self.canary
        self.scratch = self.canary.copy()

    def _alloc(self, vm, kind, size):
        if kind == "pageable":
            return np.empty(size, np.uint8)
        p = vm.PinnedBuffer(size)
        self._pinned.append(p)
        return p.array

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.src = self.dst = None
        for p in self._pinned:
            p.free()


def oracle_hashes(orc, buf, n, bb):
    lens = block_lens(n, bb)
    return lens, orc.hash_blocks(buf[:n], np.arange(lens.size, dtype=np.uint64) * bb, lens)


@functools.lru_cache(maxsize=None)
def _launches(n, bb, slot, lanes):
    return launches(block_lens(n, bb), slot, lanes)


def check_call(vm, bufs, n, bb, lens, want, prior, valid, what, slot=SLOT, lanes=1, flags=0, streams=0):
    """One vmig_migrate_buffer call over bufs.src[:n] -> bufs.dst[:n] held to the model; dst is the canary again
    afterwards."""
    h, st = vm.migrate_buffer(bufs.src[:n], bufs.dst[:n], prior, valid, gpu_mask=1, flags=flags, block_bytes=bb,
                              lanes_per_gpu=lanes, streams_per_gpu=streams)
    nb = lens.size
    surv = survivors(want, prior, valid)
    written = np.zeros_like(surv) if flags & vm.F_HASH_ONLY else surv
    bad = np.flatnonzero(h != want)
    assert bad.size == 0, f"{what}: block {bad[0]} hashes {int(h[bad[0]]):016x}, want {int(want[bad[0]]):016x}"
    check_image(bufs.dst, bufs.src, bufs.canary, written, bb, n, what, bufs.scratch)      # first: it names the block
    wbytes = int(lens[written].sum(dtype=np.uint64))
    got = {k: st[k] for k in ("blocks_total", "blocks_skipped", "bytes_h2d", "bytes_d2h", "bytes_written",
                              "kernel_launches")}
    assert got == {"blocks_total": nb, "blocks_skipped": nb - int(surv.sum()), "bytes_h2d": n, "bytes_d2h": wbytes,
                   "bytes_written": wbytes, "kernel_launches": _launches(n, bb, slot, lanes)}, (what, got)
    paint(bufs.dst, bufs.canary, written, bb, n)


def _tails(bb):
    return (0, bb - 1, 1, 31)


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("bb", BBS, ids=BB_IDS)
def test_diff_pass_writes_exactly_the_survivors(vm, orc, bb, mem):
    k = span_blocks(bb, SLOT)
    with Buffers(vm, mem, k * bb + bb + GUARD, seed=0x5C0 + bb) as bufs:
        for tail in _tails(bb):
            n = k * bb + tail
            lens, want = oracle_hashes(orc, bufs.src, n, bb)
            for name, prior, valid in families(want, lens, bb, SLOT, seed=tail):
                if tail in (1, 31) and name not in SHORT_TAIL_MASKS:
                    continue
                check_call(vm, bufs, n, bb, lens, want, prior, valid, f"{mem} bb={bb} n={n} {name}")


@pytest.mark.parametrize("mem", MEMS)
def test_hash_only_leaves_dst_untouched(vm, orc, mem):
    """VMIG_F_HASH_ONLY with a dst: nothing is copied back or written, whatever the mask; the hashes and the skip
    count still follow it."""
    bb = 65536
    n = span_blocks(bb, SLOT) * bb + 31
    with Buffers(vm, mem, n + GUARD, seed=0x4A5) as bufs:
        lens, want = oracle_hashes(orc, bufs.src, n, bb)
        for name, prior, valid in families(want, lens, bb, SLOT, seed=1):
            check_call(vm, bufs, n, bb, lens, want, prior, valid, f"{mem} hash-only {name}", flags=vm.F_HASH_ONLY)


# (id, block bytes, buffer bytes, lanes_per_gpu, streams_per_gpu).  Three lanes deal a buffer's blocks round-robin
# (one write key per block) and each lane packs its own batches; with fewer than two blocks per lane they take
# contiguous ranges instead.
OPTION_CASES = [
    ("3lanes-4K", 4096, span_blocks(4096, SLOT, 3) * 4096 + 31, 3, 0),
    ("3lanes-4M-ranges", 4 * MiB, 4 * 4 * MiB + 31, 3, 0),
    ("1stream-64K", 65536, span_blocks(65536, SLOT) * 65536 + 1, 1, 1),
    ("1stream-slot", SLOT, span_blocks(SLOT, SLOT) * SLOT + 4095, 1, 1),
]


@pytest.mark.parametrize("mem", MEMS)
@pytest.mark.parametrize("case", OPTION_CASES, ids=[c[0] for c in OPTION_CASES])
def test_diff_pass_with_lanes_and_one_stream(vm, orc, case, mem):
    cid, bb, n, lanes, streams = case
    with Buffers(vm, mem, n + GUARD, seed=0x0B7) as bufs:
        lens, want = oracle_hashes(orc, bufs.src, n, bb)
        for name, prior, valid in families(want, lens, bb, SLOT, seed=2, lanes=lanes):
            check_call(vm, bufs, n, bb, lens, want, prior, valid, f"{mem} {cid} {name}", lanes=lanes, streams=streams)


# ------------------------------------------------------------------------------------------ the minimum staging slot
SMALL_SLOT = 4 * MiB
SMALL_SLOT_MASKS = {"run_65", "batch_edges", "random_50"}


def _child_small_slot(a):
    """The engine half of test_diff_pass_at_the_minimum_slot: every case is checked here, in the child process,
    because VMIG_SLOT_MB and VMIG_SLOTS are read once per process."""
    vm = _child_vm()
    cases = 0
    try:
        for mem in MEMS:
            for bb in (4 * MiB, 4096):
                n = span_blocks(bb, SMALL_SLOT) * bb + 31
                with Buffers(vm, mem, n + GUARD, seed=0x5517) as bufs:
                    lens, want = oracle_hashes(oracle, bufs.src, n, bb)
                    for name, prior, valid in families(want, lens, bb, SMALL_SLOT, seed=3):
                        if name in SMALL_SLOT_MASKS:
                            check_call(vm, bufs, n, bb, lens, want, prior, valid, f"{mem} slot=4M bb={bb} {name}",
                                       slot=SMALL_SLOT)
                            cases += 1
        return {"cases": cases}
    finally:
        vm.shutdown()


def test_diff_pass_at_the_minimum_slot():
    """VMIG_SLOT_MB=4 VMIG_SLOTS=2: a 4 MiB block fills a slot (one block per launch), and 4 KiB blocks close their
    batch when the slot is full (1024 blocks), not at the 4096-block cap."""
    out = _run_child("_child_small_slot", {}, {"VMIG_SLOT_MB": "4", "VMIG_SLOTS": "2"}, module="test_survivors")
    assert out["cases"] == len(MEMS) * 2 * len(SMALL_SLOT_MASKS)


# ------------------------------------------------------------------------------------------ K2 on a resident batch
def test_resident_survivor_list_is_the_model(vm, orc):
    """K1 + K2 on an HBM-resident batch with ragged lengths (0 ... bb on random blocks): K2's list is np.nonzero of
    the model, in order, for every mask."""
    n, bb, seed = 4500, 4096, 0x4E5
    rng = np.random.default_rng(seed)
    r = vm.Resident(n, bb)
    try:
        r.fill(seed)
        data = orc.splitmix_bytes(seed, n * bb)
        lens = np.full(n, bb, np.uint32)
        ragged = rng.choice(n, n // 8, replace=False)
        lens[ragged] = rng.integers(0, bb + 1, ragged.size)
        lens[ragged[:2]] = (0, bb - 1)
        for b in ragged:
            r.set_len(int(b), int(lens[b]))
        want = orc.hash_blocks(data, np.arange(n, dtype=np.uint64) * bb, lens)
        for name, prior, valid in families(want, lens, bb, None, seed=4):
            r.set_prior(prior, valid)
            r.run(1)
            h, surv = r.results()
            bad = np.flatnonzero(h != want)
            assert bad.size == 0, (name, bad[:8].tolist())
            model = np.flatnonzero(survivors(want, prior, valid))
            assert surv.size == model.size and (surv == model).all(), (
                name, int(surv.size), int(model.size), np.setdiff1d(model, surv)[:8].tolist(),
                np.setdiff1d(surv, model)[:8].tolist())
    finally:
        r.close()
