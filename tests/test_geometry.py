"""Geometry tests (-m gpu): the hash kernel (K1), the survivor compaction (K2) and the engine at the batch shapes, block
sizes and process settings that the default runs (4 MiB blocks, 32 MiB staging slots) never reach.

- K1 + K2 on HBM-resident batches of every shape around the launch-geometry edges: grid = min(SMs, ceil(n/4)), the
  static first assignment of grid*32 blocks, the atomic work counter beyond it, and K2's 1024-wide tiles.
- vmig_opts.block_bytes other than 4 MiB: block tables, the planner's 4096-block batch cap inside one file, coalesced
  D2H runs of small blocks, VERIFY and restore messages, the snapshot backfill offsets.
- Settings read once per process (VMIG_SLOT_MB, VMIG_K1_PROXY_FENCE), in a child process.

Every expected value comes from the oracle (oracle/xxh64_ref.c, the literal tar pipe) or from plain numpy, never from
a second run of the engine."""
import json
import os
import stat
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from conftest import make_rich_tree
from test_gpu import ring_boundary_case

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB4M = 4 * MiB
RB = 512                                   # the smallest resident slot
BIG = 16 * MiB + 4097                      # the big file of the block-size tests: a 1-byte last block at 4 KiB
SLOT = min(max(int(os.environ.get("VMIG_SLOT_MB", "32")), 4), 1024) << 20      # the engine's staging slot
BBS = [4096, 12288, 65536, MiB + 4096, SLOT]
BB_IDS = ["4K", "12K", "64K", "1M+4K", "slot"]


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _same_survivors(got, want, what):
    assert got.size == want.size and (got == want).all(), (
        what, int(got.size), int(want.size), np.setdiff1d(want, got)[:8].tolist(), np.setdiff1d(got, want)[:8].tolist())


def _same_hashes(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, (what, bad[:8].tolist())


# ------------------------------------------------------------------------------------------ K1 + K2, resident
# 1..5 blocks (one CTA, partly idle quads), one warp +-1, the small-grid edge n = 4*SMs (114- and 132-SM parts), one K2
# tile +-1, last K2 tiles of 1, 31 and 17 elements, the static-assignment edge n = 32*SMs, and about a thousand K2 tiles
RES_N = [1, 2, 3, 4, 5, 31, 32, 33, 455, 456, 457, 527, 528, 529, 1023, 1024, 1025, 1055, 2049, 3089,
         3647, 3648, 3649, 4223, 4224, 4225, 1 << 20]
PATTERN_SMALL_N = {1, 5, 33, 457, 529}


def _resident(vm, orc, n, seed):
    """An n-block resident batch of RB-byte slots filled with SplitMix64 stream `seed`, its bytes and oracle hashes."""
    r = vm.Resident(n, RB)
    r.fill(seed)
    data = orc.splitmix_bytes(seed, n * RB)          # fill() writes the stream over the whole batch
    offs = np.arange(n, dtype=np.uint64) * RB
    return r, data, offs, orc.hash_blocks(data, offs, np.full(n, RB, np.uint32))


def _prior_patterns(h):
    """(name, prior, valid) over the true hashes h."""
    n = h.size
    i = np.arange(n)
    one = np.ones(n, np.uint8)

    def differ(mask, bit=0):
        p = h.copy()
        p[mask] ^= np.uint64(1 << bit)
        return p
    runs = ((i + 16) % 66) < 33                      # runs of 33 (each crosses a warp edge) ...
    for t in range(1024, n, 1024):                   # ... and one across every K2 tile edge
        runs[t - 16:t + 17] = True
    no_valid = one.copy()
    no_valid[(i % 7 == 3) | (i == n - 1)] = 0
    yield "none", h, one
    yield "all", differ(i >= 0), one
    yield "alternating", differ(i % 2 == 0), one
    yield "runs_of_33", differ(runs), one
    yield "first_only", differ(i == 0), one
    yield "last_only", differ(i == n - 1), one
    yield "last_tile_only", differ(i >= (n - 1) // 1024 * 1024), one
    yield "equal_hash_not_valid", h, no_valid
    yield "bit0", differ(i % 5 == 1, 0), one
    yield "bit63", differ(i % 5 == 2, 63), one


@pytest.mark.parametrize("n", RES_N)
def test_resident_hashes_and_survivors_at_every_batch_shape(vm, orc, n):
    r, _data, _offs, want = _resident(vm, orc, n, seed=0x6E0 + n)
    try:
        r.set_prior(None)
        r.run(1)
        h, surv = r.results()
        _same_hashes(h, want, "no prior")
        _same_survivors(surv, np.arange(n), "no prior: every block survives")
        if n <= 1024 and n not in PATTERN_SMALL_N:
            return
        for name, prior, valid in _prior_patterns(want):
            r.set_prior(prior, valid)
            r.run(1)
            h, surv = r.results()
            _same_hashes(h, want, name)
            _same_survivors(surv, np.nonzero(~(valid.astype(bool) & (prior == want)))[0], name)
    finally:
        r.close()


RAGGED_AT = [0, 1, 455, 456, 527, 528, 3647, 3648, 4223, 4224]


@pytest.mark.parametrize("n", [529, 4225])
def test_resident_ragged_lengths_on_the_grid_edges(vm, orc, n):
    """Blocks of 0, 1, 31, 32, 33 and RB bytes at the indices where the first assignment changes hands (c + G*(ring +
    4*quad), G = grid) and where the work counter takes over; a zero-length block whose prior is XXH64 of the empty
    input is unchanged."""
    r, data, offs, _ = _resident(vm, orc, n, seed=0xA66 + n)
    try:
        lens = np.full(n, RB, np.uint32)
        at = sorted({b for b in RAGGED_AT if b < n} | {n - 1})
        for j, b in enumerate(at):
            lens[b] = (0, 1, 31, 32, 33, RB)[j % 6]
            r.set_len(b, int(lens[b]))
        want = orc.hash_blocks(data, offs, lens)
        r.set_prior(None)
        r.run(1)
        h, surv = r.results()
        _same_hashes(h, want, "ragged")
        _same_survivors(surv, np.arange(n), "ragged, no prior")
        zero = np.nonzero(lens == 0)[0]
        assert zero.size and (want[zero] == orc.xxh64(b"")).all()
        r.set_prior(want, np.ones(n, np.uint8))
        r.run(1)
        h, surv = r.results()
        _same_hashes(h, want, "ragged, prior")
        _same_survivors(surv, np.empty(0, np.int64), "every prior equal")
        prior = want.copy()
        prior[zero] ^= np.uint64(1)
        r.set_prior(prior, np.ones(n, np.uint8))
        r.run(1)
        _, surv = r.results()
        _same_survivors(surv, zero, "zero-length blocks with another prior")
    finally:
        r.close()


# ------------------------------------------------------------------------------------------ the engine at other block sizes
def _blen(size, bb, b):
    return min(bb, size - b * bb)


def _chosen_blocks(nb):
    """Blocks 0, 4095 and 4096 (the planner closes a batch at 4096 blocks), the last one, and a run of 40."""
    run0 = nb // 3
    return sorted(b for b in {0, 4095, 4096, nb - 1} | set(range(run0, run0 + 40)) if b < nb)


def _mutate_blocks(path, blocks, bb):
    """Invert the first (up to) 8 bytes of each block in place; the file keeps its size."""
    with open(path, "r+b") as f:
        for b in blocks:
            f.seek(b * bb)
            w = bytes(x ^ 0xFF for x in f.read(8))
            f.seek(b * bb)
            f.write(w)


def _layer(orc, root):
    root.mkdir()
    make_rich_tree(root, orc)
    (root / "huge.bin").write_bytes(orc.splitmix_bytes(0x5EED, BIG).tobytes())


def _hard_linked(root, bb):
    """(blocks, bytes) a diff pass moves for hard-linked paths.  Such a destination file is never patched in place, so
    its group is written whole, once, while the table counts its blocks under every path."""
    blocks, sizes = 0, {}
    for dirpath, _, files in os.walk(root):
        for n in files:
            s = os.lstat(os.path.join(dirpath, n))
            if stat.S_ISREG(s.st_mode) and s.st_nlink > 1:
                blocks += -(-s.st_size // bb)
                sizes[s.st_ino] = s.st_size
    return blocks, sum(sizes.values())


def _table_is(orc, path, bb, root):
    entries, want = orc.block_table_of_tree(root, bb)
    t = orc.read_table(path)
    assert t["block_bytes"] == bb and t["entries"] == entries
    _same_hashes(t["hashes"], want, str(path))
    return entries, want


def _same_tree(orc, src, dst, name):
    ref = src.with_name(name)
    ref.mkdir()
    orc.ref_copy(src, ref)
    assert orc.compare_trees(ref, dst, mtime_ns=True) == []


@pytest.mark.parametrize("bb", BBS, ids=BB_IDS)
def test_tree_copy_and_diff_pass_at_block_size(vm, orc, shm_tmp, bb):
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    _layer(orc, src)
    dst.mkdir()
    st = vm.migrate_tree(src, dst, None, shm_tmp / "v1.vmig", block_bytes=bb)
    _same_tree(orc, src, dst, "ref1")
    _, want = _table_is(orc, shm_tmp / "v1.vmig", bb, src)
    assert st["blocks_total"] == want.size and st["blocks_skipped"] == 0
    vm.hash_tree(src, shm_tmp / "h.vmig", block_bytes=bb)
    _table_is(orc, shm_tmp / "h.vmig", bb, src)
    # diff pass: only the mutated blocks of huge.bin (and the hard-linked groups, never patched in place) travel
    nb = -(-BIG // bb)
    chosen = _chosen_blocks(nb)
    _mutate_blocks(src / "huge.bin", chosen, bb)
    st = vm.migrate_tree(src, dst, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig", block_bytes=bb)
    linked_blocks, linked_bytes = _hard_linked(src, bb)
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen) + linked_blocks, (st, len(chosen), linked_blocks)
    assert st["bytes_written"] == sum(_blen(BIG, bb, b) for b in chosen) + linked_bytes
    _same_tree(orc, src, dst, "ref2")
    _table_is(orc, shm_tmp / "v2.vmig", bb, src)


def _buffer_case(vm, orc, bb, pinned):
    data = orc.splitmix_bytes(0xB0F, BIG)
    if pinned:
        a, b = vm.PinnedBuffer(BIG), vm.PinnedBuffer(BIG)
        src, dst = a.array, b.array
    else:
        src, dst = np.empty(BIG, np.uint8), np.empty(BIG, np.uint8)
    try:
        src[:] = data
        dst[:] = 0
        nb = -(-BIG // bb)
        offs = np.arange(nb, dtype=np.uint64) * bb
        lens = np.array([_blen(BIG, bb, i) for i in range(nb)], np.uint32)
        h, st = vm.migrate_buffer(src, dst, block_bytes=bb)
        assert (dst == data).all() and st["blocks_total"] == nb
        _same_hashes(h, orc.hash_blocks(data, offs, lens), "copy")
        chosen = _chosen_blocks(nb)
        for i in chosen:
            src[i * bb] ^= 0xFF
        h2, st = vm.migrate_buffer(src, dst, h, np.ones(nb, np.uint8), block_bytes=bb)
        assert st["blocks_total"] - st["blocks_skipped"] == len(chosen), st
        assert st["bytes_d2h"] == int(lens[chosen].astype(np.uint64).sum())
        assert (dst == src).all()
        _same_hashes(h2, orc.hash_blocks(src, offs, lens), "diff")
    finally:
        if pinned:
            a.free(), b.free()


@pytest.mark.parametrize("bb", BBS, ids=BB_IDS)
def test_migrate_buffer_at_block_size(vm, orc, bb):
    _buffer_case(vm, orc, bb, pinned=False)


def test_migrate_pinned_buffer_at_64k(vm, orc):
    _buffer_case(vm, orc, 65536, pinned=True)


def test_three_lanes_at_4k(vm, orc, shm_tmp):
    """The lane split with 4 KiB blocks: whole files over lanes for the rich tree, the byte-range split (lanes share
    one destination file) for a tree of one file, and a diff pass on the latter."""
    bb = 4096
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    _layer(orc, src)
    dst.mkdir()
    st = vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", block_bytes=bb, lanes_per_gpu=3)
    assert st["lanes_used"] >= 3
    _same_tree(orc, src, dst, "ref")
    _table_is(orc, shm_tmp / "t.vmig", bb, src)
    one, d1 = shm_tmp / "one", shm_tmp / "d1"
    one.mkdir(), d1.mkdir()
    (one / "huge.bin").write_bytes(orc.splitmix_bytes(0x0E, BIG).tobytes())
    st = vm.migrate_tree(one, d1, None, shm_tmp / "o1.vmig", block_bytes=bb, lanes_per_gpu=3)
    assert st["lanes_used"] >= 3
    assert (d1 / "huge.bin").read_bytes() == (one / "huge.bin").read_bytes()
    _table_is(orc, shm_tmp / "o1.vmig", bb, one)
    chosen = _chosen_blocks(-(-BIG // bb))
    _mutate_blocks(one / "huge.bin", chosen, bb)
    st = vm.migrate_tree(one, d1, shm_tmp / "o1.vmig", shm_tmp / "o2.vmig", block_bytes=bb, lanes_per_gpu=3)
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen)
    assert st["bytes_written"] == sum(_blen(BIG, bb, b) for b in chosen)
    assert (d1 / "huge.bin").read_bytes() == (one / "huge.bin").read_bytes()
    _table_is(orc, shm_tmp / "o2.vmig", bb, one)


def test_verify_names_the_corrupted_block_at_64k(vm, orc, shm_tmp, monkeypatch):
    bb = 65536
    src, dst, dst2 = shm_tmp / "src", shm_tmp / "dst", shm_tmp / "dst2"
    _layer(orc, src)
    dst.mkdir(), dst2.mkdir()
    vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", flags=vm.F_VERIFY, block_bytes=bb)
    entries, _ = _table_is(orc, shm_tmp / "t.vmig", bb, src)
    first = {rel: fb for rel, _size, fb in entries}[b"huge.bin"]
    monkeypatch.setenv("VMIG_CORRUPT_BLOCK", str(first + 100))      # a table index: huge.bin's block 100
    with pytest.raises(vm.VmigError) as ei:
        vm.migrate_tree(src, dst2, None, None, flags=vm.F_VERIFY, block_bytes=bb)
    assert ei.value.code == vm.VMIG_EVERIFY and "huge.bin block 100 " in str(ei.value), ei.value


def _snapshot_source(orc, src, bb):
    src.mkdir()
    (src / "huge.bin").write_bytes(orc.splitmix_bytes(0x51, BIG).tobytes())
    (src / "same.bin").write_bytes(orc.splitmix_bytes(0x52, 3 * bb + 5).tobytes())


def test_incremental_snapshot_backfills_at_64k(vm, orc, shm_tmp):
    """A changed file's unchanged blocks are copied from the base file at 64 KiB offsets, and the increment restores
    to its source."""
    bb = 65536
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    _snapshot_source(orc, src, bb)
    v1.mkdir(), v2.mkdir()
    v1_huge = (src / "huge.bin").read_bytes()
    vm.snapshot_tree(src, v1, None, None, shm_tmp / "v1.vmig", flags=vm.F_VERIFY, block_bytes=bb)
    nb = -(-BIG // bb)
    chosen = [3, 100, 101, 102, nb - 1]
    _mutate_blocks(src / "huge.bin", chosen, bb)
    st = vm.snapshot_tree(src, v2, v1, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig", flags=vm.F_VERIFY, block_bytes=bb)
    assert st["files_linked"] == 1 and st["files_backfilled"] == 1, st
    assert st["bytes_backfilled"] == BIG - sum(_blen(BIG, bb, b) for b in chosen), st
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen)
    for name in ("huge.bin", "same.bin"):
        assert (v2 / name).read_bytes() == (src / name).read_bytes(), name
    assert (v1 / "huge.bin").read_bytes() == v1_huge                    # the base snapshot is untouched
    _table_is(orc, shm_tmp / "v2.vmig", bb, src)
    ref, dst = shm_tmp / "ref", shm_tmp / "dst"
    ref.mkdir(), dst.mkdir()
    orc.ref_copy(src, ref)
    vm.restore_tree(v2, shm_tmp / "v2.vmig", dst, block_bytes=bb)
    assert orc.compare_trees(ref, dst) == []


def test_restore_names_the_damaged_64k_block(vm, orc, shm_tmp):
    """A full snapshot at 64 KiB restores; after one byte of it at offset o rots, the restore refuses it and names
    block o // 64 KiB."""
    bb = 65536
    src, snap, ref, dst = shm_tmp / "src", shm_tmp / "snap", shm_tmp / "ref", shm_tmp / "dst"
    _snapshot_source(orc, src, bb)
    snap.mkdir(), ref.mkdir(), dst.mkdir()
    vm.snapshot_tree(src, snap, None, None, shm_tmp / "snap.vmig", flags=vm.F_VERIFY, block_bytes=bb)
    _table_is(orc, shm_tmp / "snap.vmig", bb, src)
    orc.ref_copy(src, ref)
    vm.restore_tree(snap, shm_tmp / "snap.vmig", dst, block_bytes=bb)
    assert orc.compare_trees(ref, dst) == []
    o = 77 * bb + 1234
    with open(snap / "huge.bin", "r+b") as f:
        f.seek(o)
        x = f.read(1)
        f.seek(o)
        f.write(bytes([x[0] ^ 0x5A]))
    dst2 = shm_tmp / "dst2"
    dst2.mkdir()
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(snap, shm_tmp / "snap.vmig", dst2, block_bytes=bb)
    assert ei.value.code == vm.VMIG_ECORRUPT
    assert f"huge.bin block {o // bb} " in vm.last_error(), vm.last_error()


def test_block_size_limits(vm, orc, shm_tmp):
    """A block larger than the slot or not a multiple of 4096 is refused before anything is written; a prior table
    written at another block size is refused as a table error."""
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    src.mkdir(), dst.mkdir()
    (src / "a.bin").write_bytes(orc.splitmix_bytes(0x11, 3 * 65536 + 7).tobytes())
    for bb in (SLOT + 4096, 6144):
        for call in (lambda: vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", block_bytes=bb),
                     lambda: vm.hash_tree(src, shm_tmp / "t.vmig", block_bytes=bb),
                     lambda: vm.migrate_buffer(np.zeros(8192, np.uint8), np.zeros(8192, np.uint8), block_bytes=bb)):
            with pytest.raises(vm.VmigError) as ei:
                call()
            assert ei.value.code == vm.VMIG_EINVAL, (bb, ei.value)
        assert os.listdir(dst) == [] and not (shm_tmp / "t.vmig").exists()
    other = shm_tmp / "other"
    other.mkdir()
    vm.migrate_tree(src, other, None, shm_tmp / "t64.vmig", block_bytes=65536)
    with pytest.raises(vm.VmigError) as ei:
        vm.migrate_tree(src, dst, shm_tmp / "t64.vmig", shm_tmp / "t.vmig", block_bytes=4096)
    assert ei.value.code == vm.VMIG_ETABLE
    assert os.listdir(dst) == [] and not (shm_tmp / "t.vmig").exists()


# ------------------------------------------------------------------------------------------ settings read once per process
def _run_child(fn: str, arg: dict, env: dict, module: str = "test_geometry") -> dict:
    """Run <module>.<fn>(arg) in a new Python process with `env` added; it prints one JSON line of results."""
    here = Path(__file__).resolve().parent
    code = ("import importlib, json, sys; sys.path[:0] = sys.argv[1:3]; t = importlib.import_module(sys.argv[5]); "
            "print(json.dumps(getattr(t, sys.argv[3])(json.loads(sys.argv[4]))))")
    r = subprocess.run([sys.executable, "-c", code, str(here), str(here.parent), fn, json.dumps(arg), module],
                       env={**os.environ, **env}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _child_vm():
    import __graft_entry__ as g
    vm = g.load_pkg()
    vm.init(0)
    return vm


def _child_small_slot(a):
    """The engine half of test_minimum_slot_one_block_per_launch."""
    vm = _child_vm()
    try:
        out = {"copy": vm.migrate_tree(a["src"], a["dst"], None, a["t1"])}
        _mutate_blocks(Path(a["src"]) / "huge.bin", a["mutate"], BB4M)
        out["diff"] = vm.migrate_tree(a["src"], a["dst"], a["t1"], a["t2"])
        out["whole"] = vm.migrate_tree(a["whole"], a["whole_dst"], None, a["t3"])
        buf = np.fromfile(a["one_block"], np.uint8)
        out["one_block"] = [str(int(x)) for x in vm.hash_blocks(buf, [0], [buf.size])[0]]
        try:
            vm.hash_blocks(np.zeros(BB4M + 1, np.uint8), [0], [BB4M + 1])
            out["over_slot"] = 0
        except vm.VmigError as e:
            out["over_slot"] = e.code
        return out
    finally:
        vm.shutdown()


def test_minimum_slot_one_block_per_launch(vm, orc, shm_tmp):
    """VMIG_SLOT_MB=4 VMIG_SLOTS=2: each 4 MiB block fills a slot, so every batch is a one-block K1 launch on a grid of
    one; a tree copy, a diff pass and K1 direct still give the oracle's answers, and a block one byte over is
    refused."""
    src, dst, whole, whole_dst = shm_tmp / "src", shm_tmp / "dst", shm_tmp / "whole", shm_tmp / "whole_dst"
    _layer(orc, src)
    dst.mkdir(), whole.mkdir(), whole_dst.mkdir()
    for i, k in enumerate((1, 2, 3)):
        (whole / f"w{k}.bin").write_bytes(orc.splitmix_bytes(0x40 + i, k * BB4M).tobytes())
    entries1, want1 = orc.block_table_of_tree(src)
    mutate = [1, 4]
    out = _run_child("_child_small_slot", {
        "src": str(src), "dst": str(dst), "t1": str(shm_tmp / "t1.vmig"), "t2": str(shm_tmp / "t2.vmig"),
        "mutate": mutate, "whole": str(whole), "whole_dst": str(whole_dst), "t3": str(shm_tmp / "t3.vmig"),
        "one_block": str(whole / "w1.bin")}, {"VMIG_SLOT_MB": "4", "VMIG_SLOTS": "2"})
    t1 = orc.read_table(shm_tmp / "t1.vmig")
    assert t1["entries"] == entries1
    _same_hashes(t1["hashes"], want1, "copy")
    assert out["copy"]["blocks_total"] == want1.size
    linked_blocks, linked_bytes = _hard_linked(src, BB4M)
    assert out["diff"]["blocks_total"] - out["diff"]["blocks_skipped"] == len(mutate) + linked_blocks, out["diff"]
    assert out["diff"]["bytes_written"] == sum(_blen(BIG, BB4M, b) for b in mutate) + linked_bytes
    _same_tree(orc, src, dst, "ref2")
    _table_is(orc, shm_tmp / "t2.vmig", BB4M, src)
    assert out["whole"]["blocks_total"] == 6 and out["whole"]["kernel_launches"] == 6, out["whole"]
    assert orc.compare_trees(whole, whole_dst, ignore_root_mtime=True) == []
    _table_is(orc, shm_tmp / "t3.vmig", BB4M, whole)
    assert [int(x) for x in out["one_block"]] == orc.hash_file(whole / "w1.bin").tolist()
    assert out["over_slot"] == vm.VMIG_EINVAL


FENCE_N, FENCE_BB, FENCE_SEED = 2048, 128 * 1024 + 512, 0xFE5CE


def _child_proxy_fence(a):
    """The engine half of test_proxy_fence_variant_equals_the_oracle."""
    vm = _child_vm()
    try:
        buf, offs, lens = ring_boundary_case()
        ring = vm.hash_blocks(buf, offs, lens)[0]
        r = vm.Resident(FENCE_N, FENCE_BB)
        try:
            r.fill(FENCE_SEED)
            r.set_prior(None)
            r.run(1)
            h, surv = r.results()
        finally:
            r.close()
        return {"ring": [str(int(x)) for x in ring], "resident": [str(int(x)) for x in h], "survivors": int(surv.size)}
    finally:
        vm.shutdown()


def test_proxy_fence_variant_equals_the_oracle(vm, orc):
    """VMIG_K1_PROXY_FENCE=1 (a fence.proxy.async before each stage is handed to the chains) computes the same hashes
    as the default variant does, bit for bit: the ring-boundary length set and a 2 048-block resident pass."""
    out = _run_child("_child_proxy_fence", {}, {"VMIG_K1_PROXY_FENCE": "1"})
    buf, offs, lens = ring_boundary_case()
    _same_hashes(np.array([int(x) for x in out["ring"]], np.uint64), orc.hash_blocks(buf, offs, lens), "ring lengths")
    data = orc.splitmix_bytes(FENCE_SEED, FENCE_N * FENCE_BB)
    want = orc.hash_blocks(data, np.arange(FENCE_N, dtype=np.uint64) * FENCE_BB, np.full(FENCE_N, FENCE_BB, np.uint32))
    _same_hashes(np.array([int(x) for x in out["resident"]], np.uint64), want, "resident")
    assert out["survivors"] == FENCE_N
