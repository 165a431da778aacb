"""Offsets past 4 GiB on the GPU (-m gpu): one host buffer, one file and one snapshot backfill longer than 2^32 bytes.

Block lengths, slot offsets and file indices are 32-bit by design; file offsets, buffer offsets and run lengths are
64-bit.  A truncated offset does not crash: it puts the right bytes in the wrong place, or hashes the wrong range and
finds a block unchanged.  So the sources here are sparse (holes on tmpfs, untouched pages in memory) with SplitMix64
islands where a truncation would show: the first blocks, either side of 2^32, the 2 GiB and 3 GiB regions and the tail.
A destination is all hole or all zero wherever nothing should have been written.

The byte-range lane split of a one-file tree lives in csrc/vmig_api.cu (run_blocks), not in the CUDA-free planner, so it
is covered here and not in tests/plan_unit.cpp.

Every expected value comes from the oracle (oracle/xxh64_ref.c, the table reader, compare_trees) or from plain numpy,
never from a second run of the engine.  Each phase deletes what it no longer needs; the peak is about 9 GiB, of tmpfs in
the tree tests and of page-locked memory in the pinned one, and the module skips unless 14 GiB are free."""
import json
import os
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
G4 = 1 << 32
BB4M = 4 * MiB
BB_ODD = MiB + 4096                        # one block straddles 2^32
BIGF = G4 + 9 * MiB + 777
NEED = 14 << 30
KAT = json.loads((Path(__file__).parent / "golden" / "xxh64_kat.json").read_text())
# (start, length) of the data islands; everything else is zero
ISLANDS = [(0, 9 * MiB), (2 << 30, 5 * MiB), ((3 << 30) - MiB, 6 * MiB), (G4 - 9 * MiB, BIGF - (G4 - 9 * MiB))]


def _free_bytes(p) -> int:
    st = os.statvfs(p)
    avail = [st.f_bavail * st.f_frsize]
    for line in Path("/proc/meminfo").read_text().splitlines():
        if line.startswith("MemAvailable:"):
            avail.append(int(line.split()[1]) * 1024)
    return min(avail)


@pytest.fixture(scope="module", autouse=True)
def _gpu_and_room(vm):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else "/tmp"
    free = _free_bytes(base)
    if free < NEED:
        pytest.skip(f"needs {NEED >> 30} GiB free in {base} and in MemAvailable for files and buffers past 4 GiB; {free >> 30} GiB are free")
    vm.init(0)
    yield
    vm.shutdown()


def _blen(size, bb, i):
    return min(bb, size - i * bb)


def _same_hashes(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, (what, bad[:8].tolist())


def _island_bytes(orc, seed, k):
    start, n = ISLANDS[k]
    return orc.splitmix_bytes(seed + k, n)


def _fill_buffer(orc, buf, seed):
    for k, (start, n) in enumerate(ISLANDS):
        buf[start:start + n] = _island_bytes(orc, seed, k)


def _sparse_file(orc, path, seed):
    with open(path, "wb") as f:
        f.truncate(BIGF)
        for k, (start, n) in enumerate(ISLANDS):
            f.seek(start)
            f.write(_island_bytes(orc, seed, k).tobytes())
    assert os.path.getsize(path) == BIGF


def _tree(orc, root, seed=0x1A):
    root.mkdir()
    (root / "a.bin").write_bytes(orc.splitmix_bytes(seed + 100, 2 * BB4M + 5).tobytes())
    _sparse_file(orc, root / "huge.bin", seed)
    (root / "z.bin").write_bytes(orc.splitmix_bytes(seed + 101, 70000).tobytes())


def _mutate_file(path, blocks, bb):
    """Flip the first 8 bytes of each block."""
    with open(path, "r+b") as f:
        for b in blocks:
            f.seek(b * bb)
            n = min(8, BIGF - b * bb)
            x = f.read(n)
            f.seek(b * bb)
            f.write(bytes(c ^ 0xFF for c in x))


def _table_is(orc, path, bb, root):
    entries, want = orc.block_table_of_tree(root, bb)
    t = orc.read_table(path)
    assert t["block_bytes"] == bb and t["entries"] == entries
    _same_hashes(t["hashes"], want, str(path))
    return entries, want


def _same_file(orc, a, b, bb=BB4M):
    assert os.path.getsize(a) == os.path.getsize(b) == BIGF
    _same_hashes(orc.hash_file(a, bb), orc.hash_file(b, bb), f"{a} vs {b}")


def _first_block_of(entries, rel):
    return {r: fb for r, _size, fb in entries}[rel]


# ------------------------------------------------------------------------------------------ K1 direct
def test_hash_blocks_either_side_of_4GiB(vm, orc):
    buf = np.zeros(BIGF, np.uint8)
    _fill_buffer(orc, buf, 0x71)
    L = BB4M
    blocks = [(G4 - L, L),                 # ends at 2^32
              (G4 - 1 - L, L),             # ends at 2^32 - 1
              (G4 - 1, L), (G4, L), (G4 + 1, L),
              (G4 - MiB - 3, 2 * MiB + 7),  # straddles
              (G4 - 1, 1), (G4 - 1, 2), (G4, 1),
              (BIGF - 777, 777), (BIGF - L, L),
              (0, L), (3, 65537), (4 * MiB, 4 * MiB), (2 << 30, L), ((2 << 30) + 4096 - 1, 4097), (3 << 30, MiB + 1),
              (1 << 30, L)]                # a hole
    order = np.random.default_rng(0x4A).permutation(len(blocks))
    offs = np.array([blocks[i][0] for i in order], np.uint64)
    lens = np.array([blocks[i][1] for i in order], np.uint32)
    got, _ms = vm.hash_blocks(buf, offs, lens)
    _same_hashes(got, orc.hash_blocks(buf, offs, lens), "K1 around 2^32")
    assert int(got[list(order).index(len(blocks) - 1)]) == int(KAT["zeros_4MiB"], 16)


# ------------------------------------------------------------------------------------------ host buffers
def _nonzero_total(a):
    return sum(int(np.count_nonzero(a[o:o + 64 * MiB])) for o in range(0, a.size, 64 * MiB))


def _buffer_case(vm, orc, bb, src, dst):
    """src and dst are BIGF bytes; dst is all zero."""
    _fill_buffer(orc, src, 0xB0 + (bb >> 12))
    nb = -(-BIGF // bb)
    offs = np.arange(nb, dtype=np.uint64) * np.uint64(bb)
    lens = np.full(nb, bb, np.uint32)
    lens[-1] = BIGF - (nb - 1) * bb
    want = orc.hash_blocks(src, offs, lens)
    h, st = vm.migrate_buffer(src, None, flags=vm.F_HASH_ONLY, block_bytes=bb)
    assert st["bytes_total"] == BIGF and st["blocks_total"] == nb
    _same_hashes(h, want, "hash-only pass")
    i0 = G4 // bb                                       # the block that holds offset 2^32 (it starts there at 4 MiB and 64 KiB)
    chosen = sorted({i0 - 1, i0, min(i0 + 3, nb - 1), nb - 1})
    assert (i0 * bb < G4) == (bb == BB_ODD)
    for i in chosen:
        src[i * bb] ^= 0xFF
    h2, st = vm.migrate_buffer(src, dst, want, np.ones(nb, np.uint8), block_bytes=bb)
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen), st
    assert st["bytes_d2h"] == sum(int(lens[i]) for i in chosen), st
    moved = 0
    for i in chosen:
        a, b = i * bb, i * bb + int(lens[i])
        assert (dst[a:b] == src[a:b]).all(), (bb, i)
        moved += int(np.count_nonzero(src[a:b]))
        for lo, hi in ((max(a - 2 * bb, 0), a), (b, min(b + 2 * bb, BIGF))):          # the two blocks either side
            if not any(lo <= j * bb < hi for j in chosen):
                assert not dst[lo:hi].any(), (bb, i, lo)
    assert moved > sum(int(lens[i]) for i in chosen) * 0.99                             # the ranges hold data, not zeros
    assert _nonzero_total(dst) == moved                                                 # and nothing else was written
    want2 = want.copy()
    sel = np.array(chosen)
    want2[sel] = orc.hash_blocks(src, offs[sel], lens[sel])
    assert (want2[sel] != want[sel]).all()
    _same_hashes(h2, want2, "diff pass")


@pytest.mark.parametrize("bb", [BB4M, BB_ODD, 65536], ids=["4M", "1M+4K", "64K"])
def test_migrate_buffer_past_4GiB(vm, orc, bb):
    _buffer_case(vm, orc, bb, np.zeros(BIGF, np.uint8), np.zeros(BIGF, np.uint8))


def test_migrate_pinned_buffer_past_4GiB(vm, orc):
    bufs = []
    try:
        try:
            for _ in range(2):
                bufs.append(vm.PinnedBuffer(BIGF))
        except vm.VmigError as e:
            pytest.skip(f"test_migrate_pinned_buffer_past_4GiB: no {BIGF >> 20} MiB of page-locked memory twice ({e})")
        for b in bufs:
            b.array[:] = 0
        _buffer_case(vm, orc, BB4M, bufs[0].array, bufs[1].array)
    finally:
        for b in bufs:
            b.free()


# ------------------------------------------------------------------------------------------ trees
def test_tree_copy_and_diff_pass_of_a_file_past_4GiB(vm, orc, shm_tmp):
    bb = BB4M
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    _tree(orc, src)
    dst.mkdir()
    vm.hash_tree(src, shm_tmp / "h.vmig")
    entries, want = _table_is(orc, shm_tmp / "h.vmig", bb, src)
    fb = _first_block_of(entries, b"huge.bin")
    assert int(want[fb + 256]) == int(KAT["zeros_4MiB"], 16)                  # a hole hashes as zeros
    st = vm.migrate_tree(src, dst, None, shm_tmp / "v1.vmig", flags=vm.F_VERIFY)
    assert st["bytes_total"] == sum(s for _r, s, _f in entries) and st["blocks_total"] == want.size and st["blocks_skipped"] == 0
    assert st["bytes_written"] == st["bytes_total"]
    t1 = orc.read_table(shm_tmp / "v1.vmig")
    assert t1["entries"] == entries
    _same_hashes(t1["hashes"], want, "copy")
    _same_file(orc, src / "huge.bin", dst / "huge.bin")
    assert orc.compare_trees(src, dst, content=False) == []
    for n in ("a.bin", "z.bin"):
        assert (dst / n).read_bytes() == (src / n).read_bytes()
    # diff pass in place
    nb = -(-BIGF // bb)
    chosen = [G4 // bb - 1, G4 // bb, nb - 1]
    _mutate_file(src / "huge.bin", chosen, bb)
    st = vm.migrate_tree(src, dst, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig", flags=vm.F_VERIFY)
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen), st
    assert st["bytes_written"] == sum(_blen(BIGF, bb, b) for b in chosen), st
    _same_file(orc, src / "huge.bin", dst / "huge.bin")
    _, want2 = _table_is(orc, shm_tmp / "v2.vmig", bb, src)
    assert sorted(np.nonzero(want2 != want)[0].tolist()) == [fb + b for b in chosen]


def test_three_lanes_share_one_file_past_4GiB(vm, orc, shm_tmp):
    """One file and three lanes: the block list is cut into byte ranges of about 1.43 GiB, the last of which holds
    offset 2^32; at 1 MiB + 4096 one block straddles it."""
    bb = BB_ODD
    one, d1 = shm_tmp / "one", shm_tmp / "d1"
    one.mkdir(), d1.mkdir()
    _sparse_file(orc, one / "huge.bin", 0x3C)
    st = vm.migrate_tree(one, d1, None, shm_tmp / "o1.vmig", block_bytes=bb, lanes_per_gpu=3)
    assert st["lanes_used"] >= 3 and st["bytes_written"] == BIGF
    _, want = _table_is(orc, shm_tmp / "o1.vmig", bb, one)
    _same_file(orc, one / "huge.bin", d1 / "huge.bin", bb)
    nb = -(-BIGF // bb)
    chosen = [1, (2 << 30) // bb + 1, G4 // bb, nb - 1]           # one in each lane's range: near 0, 2 GiB, and past 2^32
    assert chosen[2] * bb < G4 < (chosen[2] + 1) * bb
    _mutate_file(one / "huge.bin", chosen, bb)
    st = vm.migrate_tree(one, d1, shm_tmp / "o1.vmig", shm_tmp / "o2.vmig", block_bytes=bb, lanes_per_gpu=3)
    assert st["lanes_used"] >= 3
    assert st["blocks_total"] - st["blocks_skipped"] == len(chosen), st
    assert st["bytes_written"] == sum(_blen(BIGF, bb, b) for b in chosen), st
    _same_file(orc, one / "huge.bin", d1 / "huge.bin", bb)
    _, want2 = _table_is(orc, shm_tmp / "o2.vmig", bb, one)
    assert np.nonzero(want2 != want)[0].tolist() == chosen


def test_verify_names_a_block_past_4GiB(vm, orc, shm_tmp, monkeypatch):
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    _tree(orc, src)
    dst.mkdir()
    n = G4 // BB4M + 1                                             # huge.bin's block 1025, at offset 2^32 + 4 MiB
    a_blocks = -(-os.path.getsize(src / "a.bin") // BB4M)
    monkeypatch.setenv("VMIG_CORRUPT_BLOCK", str(a_blocks + n))    # a table index
    with pytest.raises(vm.VmigError) as ei:
        vm.migrate_tree(src, dst, None, None, flags=vm.F_VERIFY)
    assert ei.value.code == vm.VMIG_EVERIFY and f"huge.bin block {n} " in str(ei.value), ei.value
    # the flipped bit is where the message says, and nowhere else
    got, want = orc.hash_file(dst / "huge.bin"), orc.hash_file(src / "huge.bin")
    assert np.nonzero(got != want)[0].tolist() == [n]


# ------------------------------------------------------------------------------------------ snapshots, restore, scrub
def _flip(path, o):
    with open(path, "r+b") as f:
        f.seek(o)
        x = f.read(1)
        f.seek(o)
        f.write(bytes([x[0] ^ 0x5A]))


def test_snapshot_backfill_of_more_than_4GiB(vm, orc, shm_tmp):
    bb = BB4M
    src, v1, v2, v3 = (shm_tmp / n for n in ("src", "v1", "v2", "v3"))
    _tree(orc, src, seed=0x5A)
    for d in (v1, v2, v3):
        d.mkdir()
    nb = -(-BIGF // bb)
    last_len = _blen(BIGF, bb, nb - 1)
    vm.snapshot_tree(src, v1, None, None, shm_tmp / "v1.vmig", flags=vm.F_VERIFY)
    _table_is(orc, shm_tmp / "v1.vmig", bb, src)
    v1_huge = orc.hash_file(v1 / "huge.bin")
    _same_hashes(v1_huge, orc.hash_file(src / "huge.bin"), "full snapshot")
    # only the last block changes: everything before it is one backfill of more than 2^32 bytes
    _mutate_file(src / "huge.bin", [nb - 1], bb)
    st = vm.snapshot_tree(src, v2, v1, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig", flags=vm.F_VERIFY)
    assert st["files_linked"] == 2 and st["files_backfilled"] == 1, st
    assert st["bytes_backfilled"] == BIGF - last_len and st["bytes_backfilled"] > G4, st
    assert st["blocks_total"] - st["blocks_skipped"] == 1 and st["bytes_written"] == last_len, st
    _same_file(orc, src / "huge.bin", v2 / "huge.bin")
    _table_is(orc, shm_tmp / "v2.vmig", bb, src)
    _same_hashes(orc.hash_file(v1 / "huge.bin"), v1_huge, "the base snapshot is untouched")
    assert os.stat(v2 / "huge.bin").st_ino != os.stat(v1 / "huge.bin").st_ino
    os.unlink(v1 / "huge.bin")                                     # v2 shares a.bin and z.bin with v1: those stay as they are
    # renamed, and its first block changed: the rest is found under the old path
    os.rename(src / "huge.bin", src / "moved.bin")
    _mutate_file(src / "moved.bin", [0], bb)
    st = vm.snapshot_tree(src, v3, v2, shm_tmp / "v2.vmig", shm_tmp / "v3.vmig", flags=vm.F_VERIFY)
    assert st["files_linked"] == 2 and st["files_backfilled"] == 1, st
    assert st["bytes_backfilled"] == BIGF - bb and st["bytes_written"] == bb, st
    _same_file(orc, src / "moved.bin", v3 / "moved.bin")
    _table_is(orc, shm_tmp / "v3.vmig", bb, src)
    assert not (v3 / "huge.bin").exists()
    os.unlink(v2 / "huge.bin")
    # the increment restores to its source
    dst = shm_tmp / "dst"
    dst.mkdir()
    vm.restore_tree(v3, shm_tmp / "v3.vmig", dst)
    _same_file(orc, src / "moved.bin", dst / "moved.bin")
    assert orc.compare_trees(src, dst, content=False, ignore_root_mtime=True) == []


def test_restore_and_scrub_name_a_damaged_block_past_4GiB(vm, orc, shm_tmp):
    bb = BB4M
    src, v1, v2, dst = (shm_tmp / n for n in ("src", "v1", "v2", "dst"))
    _tree(orc, src, seed=0x6B)
    for d in (v1, v2, dst):
        d.mkdir()
    vm.snapshot_tree(src, v1, None, None, shm_tmp / "v1.vmig")
    os.unlink(src / "z.bin")
    st = vm.snapshot_tree(src, v2, v1, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig")
    assert st["files_backfilled"] == 0 and st["bytes_written"] == 0, st
    ino = os.stat(v1 / "huge.bin").st_ino
    assert os.stat(v2 / "huge.bin").st_ino == ino                  # the two versions share the file
    pairs = [(v1, shm_tmp / "v1.vmig"), (v2, shm_tmp / "v2.vmig")]
    r = vm.scrub_store(pairs, shm_tmp / "scrub0.txt")
    assert r["verdicts"] == [vm.VMIG_OK] * 2 and r["findings"] == []
    assert r["bytes_unique"] == sum(os.path.getsize(v1 / n) for n in ("a.bin", "huge.bin", "z.bin")) and r["bytes_unique"] > G4
    assert r["bytes_referenced"] == 2 * BIGF + 2 * os.path.getsize(v1 / "a.bin") + os.path.getsize(v1 / "z.bin")
    o = G4 + 5 * MiB + 123
    _flip(v1 / "huge.bin", o)
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(v2, shm_tmp / "v2.vmig", dst)
    assert ei.value.code == vm.VMIG_ECORRUPT
    assert f"huge.bin block {o // bb} " in vm.last_error(), vm.last_error()
    r = vm.scrub_store(pairs, shm_tmp / "scrub1.txt")
    assert r["verdicts"] == [vm.VMIG_ECORRUPT] * 2
    assert [(f["version"], f["kind"], f["path"], f["block"]) for f in r["findings"]] == [
        (0, "block", "huge.bin", o // bb), (1, "block", "huge.bin", o // bb)]
    want = orc.hash_file(src / "huge.bin")
    got = orc.hash_file(v1 / "huge.bin")
    assert np.nonzero(got != want)[0].tolist() == [o // bb]
    assert all(f["want"] == int(want[o // bb]) and f["got"] == int(got[o // bb]) for f in r["findings"])
    assert r["blocks_damaged"] == 1 and r["files_damaged"] == 2 and r["versions_damaged"] == 2
