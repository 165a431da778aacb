"""vmig_restore_tree on the GPU (-m gpu): a snapshot is restored only while it still matches its block table.

Clean restores must equal the reference's tar copy of the snapshot and report what vmig_migrate_tree reports; a
snapshot that lost, gained or resized a file is refused before the destination is touched; a changed block is found
by the hash the GPU computes anyway, and is never written."""
import os
import shutil
from pathlib import Path

import pytest

from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB = 4 * MiB
# counters, not timings: what a restore of an intact snapshot must report exactly like a migration
COUNTERS = ("bytes_total", "bytes_h2d", "bytes_d2h", "bytes_written", "blocks_total", "blocks_skipped", "files", "dirs",
            "symlinks", "hardlinks", "specials", "kernel_launches", "gpus_used", "lanes_used", "pruned", "files_untrusted")


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _handoff(vm):
    import importlib
    return importlib.import_module(vm.__name__ + ".handoff")


def _snapshot(vm, orc, base: Path, multi: int = 3 * BB + 4097):
    """A version snapshot as SnapshotVersion leaves it: the rich tree plus a multi-block file, copied by the engine into
    base/snap with its block table base/snap.vmig."""
    src, snap = base / "src", base / "snap"
    src.mkdir(), snap.mkdir()
    make_rich_tree(src, orc)
    (src / "multi.bin").write_bytes(orc.splitmix_bytes(77, multi).tobytes())
    vm.migrate_tree(src, snap, None, base / "snap.vmig", flags=vm.F_VERIFY)
    return snap, base / "snap.vmig"


def _flip(path: Path, off: int) -> bytes:
    """XOR one byte of the file in place; returns the byte that was there."""
    with open(path, "r+b") as f:
        f.seek(off)
        old = f.read(1)
        f.seek(off)
        f.write(bytes([old[0] ^ 0x5A]))
    return old


def _state(root: Path) -> dict:
    """Every entry under root with its kind, content and mtime: what 'untouched' means."""
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for n in [""] + dirnames + filenames:
            p = os.path.join(dirpath, n) if n else dirpath
            st = os.lstat(p)
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[os.path.relpath(p, root)] = (st.st_mode, st.st_mtime_ns, st.st_size if body is not None else 0, body)
    return out


def _prepopulated(base: Path) -> Path:
    dst = base / "dst"
    (dst / "sub").mkdir(parents=True)
    (dst / "stale.bin").write_bytes(b"s" * 5000)          # not in the snapshot: VMIG_F_PRUNE would remove it
    (dst / "sub" / "small.txt").write_bytes(b"old")
    (dst / "multi.bin").write_bytes(b"m" * 10000)
    os.symlink("stale.bin", dst / "lnk_old")
    for p in (dst / "stale.bin", dst / "sub" / "small.txt", dst / "multi.bin", dst / "sub", dst):
        os.utime(p, ns=(1_500_000_000_000_000_000, 1_500_000_000_000_000_000))
    return dst


def _expect_corrupt(vm, call, *needles):
    with pytest.raises(vm.VmigError) as ei:
        call()
    assert ei.value.code == vm.VMIG_ECORRUPT, ei.value
    for n in needles:
        assert n in str(ei.value), (n, str(ei.value))
    return str(ei.value)


# ------------------------------------------------------------------------------------------ clean restore
def test_clean_restore_equals_tar_copy_and_reports_like_migrate(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst, ref, dst2 = shm_tmp / "dst", shm_tmp / "ref", shm_tmp / "dst2"
    dst.mkdir(), ref.mkdir(), dst2.mkdir()
    st = vm.restore_tree(snap, table, dst, None, shm_tmp / "out.vmig")
    orc.ref_copy(snap, ref)
    assert orc.compare_trees(ref, dst) == []
    _, want = orc.block_table_of_tree(snap)
    assert (vm.table_hashes(shm_tmp / "out.vmig") == want).all()
    st2 = vm.migrate_tree(snap, dst2, None, shm_tmp / "out2.vmig")
    assert {k: st[k] for k in COUNTERS} == {k: st2[k] for k in COUNTERS}
    assert st["hardlinks"] == 2 and st["specials"] >= 1 and st["symlinks"] == 2


# ------------------------------------------------------------------------------------------ a changed block
@pytest.mark.parametrize("lanes", [1, 3])
def test_flipped_byte_in_block_k_is_never_written(vm, orc, shm_tmp, lanes):
    snap, table = _snapshot(vm, orc, shm_tmp)
    k = 2
    _flip(snap / "multi.bin", k * BB + 12345)
    bad = (snap / "multi.bin").read_bytes()[k * BB:(k + 1) * BB]
    dst = shm_tmp / "dst"
    dst.mkdir()
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, dst, None, shm_tmp / "out.vmig", lanes_per_gpu=lanes),
                    f"multi.bin block {k} ")
    assert not (shm_tmp / "out.vmig").exists()
    if (dst / "multi.bin").exists():
        assert (dst / "multi.bin").read_bytes()[k * BB:(k + 1) * BB] != bad


# ------------------------------------------------------------------------------------------ plan-time refusals
@pytest.mark.parametrize("case", ["deleted", "added", "truncated"])
def test_tree_that_is_not_the_tables_leaves_the_destination_untouched(vm, orc, shm_tmp, case):
    snap, table = _snapshot(vm, orc, shm_tmp)
    if case == "deleted":
        os.unlink(snap / "exact.bin")
        needles = ("exact.bin", "missing")
    elif case == "added":
        (snap / "sub" / "new.txt").write_bytes(b"new")
        needles = ("sub/new.txt", "extra")
    else:
        with open(snap / "multi.bin", "r+b") as f:
            f.truncate((snap / "multi.bin").stat().st_size - 1)
        needles = ("multi.bin", "resized")
    dst = _prepopulated(shm_tmp)
    before = _state(dst)
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, dst, None, shm_tmp / "out.vmig",
                                                flags=vm.F_PRUNE | vm.F_VERIFY), *needles)
    assert _state(dst) == before
    assert not (shm_tmp / "out.vmig").exists()


def test_snapshot_without_its_table_is_refused(vm, orc, shm_tmp):
    """A SnapshotVersion that failed part way: a short diff/ and no blocks.vmig."""
    snap, table = _snapshot(vm, orc, shm_tmp)
    os.unlink(table)
    with open(snap / "multi.bin", "r+b") as f:
        f.truncate(BB)
    dst = _prepopulated(shm_tmp)
    before = _state(dst)
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(snap, table, dst, None, None, flags=vm.F_PRUNE | vm.F_VERIFY)
    assert ei.value.code == vm.VMIG_ETABLE, ei.value
    assert _state(dst) == before


# ------------------------------------------------------------------------------------------ seeded rollback
def test_seeded_rollback_moves_only_differing_blocks_and_skips_hide_nothing(vm, orc, shm_tmp):
    src, snap, v3, up = (shm_tmp / n for n in ("src", "snap", "v3", "upper"))
    for d in (src, snap, v3, up):
        d.mkdir()
    for i in range(6):
        (src / f"g{i}.bin").write_bytes(orc.splitmix_bytes(900 + i, 9 * MiB + i).tobytes())
    table = shm_tmp / "snap.vmig"
    vm.migrate_tree(src, snap, None, table, flags=vm.F_VERIFY)          # version 2 and its table
    vm.migrate_tree(snap, up, None, shm_tmp / "seed2.vmig")              # the layer holds version 2 ...
    orc.ref_copy(snap, v3)
    _flip(v3 / "g1.bin", 1 * BB + 9)
    _flip(v3 / "g4.bin", 2 * BB + 100)
    vm.migrate_tree(v3, up, shm_tmp / "seed2.vmig", shm_tmp / "seed3.vmig")   # ... then version 3: two blocks differ
    st = vm.restore_tree(snap, table, up, shm_tmp / "seed3.vmig", shm_tmp / "back.vmig", flags=vm.F_VERIFY | vm.F_PRUNE)
    assert st["files_untrusted"] == 0 and st["blocks_total"] - st["blocks_skipped"] == 2, st
    assert orc.compare_trees(snap, up) == []
    assert (vm.table_hashes(shm_tmp / "back.vmig") == vm.table_hashes(table)).all()

    # the snapshot rots; a layer filled FROM the rotten snapshot holds the same bytes, so its seed table marks the
    # block as already there -- the skip must not hide the difference from the snapshot's own table
    k = 1
    _flip(snap / "g3.bin", k * BB + 77)
    rotten = shm_tmp / "rotten"
    rotten.mkdir()
    vm.migrate_tree(snap, rotten, None, shm_tmp / "rotten.vmig")
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, rotten, shm_tmp / "rotten.vmig", shm_tmp / "r2.vmig",
                                                flags=vm.F_VERIFY | vm.F_PRUNE), f"g3.bin block {k} ")
    assert not (shm_tmp / "r2.vmig").exists()


# ------------------------------------------------------------------------------------------ hard links
def test_hard_link_swapped_in_after_the_table_is_refused_before_linking(vm, orc, shm_tmp):
    snap = shm_tmp / "snap"
    snap.mkdir()
    (snap / "a").write_bytes(orc.splitmix_bytes(1, BB + 3).tobytes())
    (snap / "b").write_bytes(orc.splitmix_bytes(2, BB + 3).tobytes())
    (snap / "c").write_bytes(b"c" * 100)
    vm.hash_tree(snap, shm_tmp / "t.vmig")
    os.unlink(snap / "b")
    os.link(snap / "a", snap / "b")
    dst = shm_tmp / "dst"
    dst.mkdir()
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, shm_tmp / "t.vmig", dst), "b block 0", "hard link")
    assert not (dst / "b").exists()


# ------------------------------------------------------------------------------------------ check-only
def test_check_only_mode_writes_nothing(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    before = sorted(os.listdir(shm_tmp))
    snap_state = _state(snap)
    st = vm.restore_tree(snap, table, None, flags=vm.F_HASH_ONLY)
    assert st["bytes_written"] == 0 and st["blocks_total"] == vm.table_info(table)["n_blocks"]
    assert sorted(os.listdir(shm_tmp)) == before and _state(snap) == snap_state
    _flip(snap / "big.bin", 2 * BB + 5)
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, None, flags=vm.F_HASH_ONLY), "big.bin block 2 ")
    assert sorted(os.listdir(shm_tmp)) == before


# ------------------------------------------------------------------------------------------ argument errors
def test_argument_errors(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst = shm_tmp / "dst"
    dst.mkdir()
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(snap, table, dst, flags=vm.F_MOVE_SRC)
    assert ei.value.code == vm.VMIG_EINVAL
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(snap, table, dst, block_bytes=1 * MiB)
    assert ei.value.code == vm.VMIG_ETABLE
    assert os.listdir(dst) == [] and (snap / "multi.bin").exists()


# ------------------------------------------------------------------------------------------ O_DIRECT
def test_flipped_block_found_with_direct_io_on_disk(vm, orc, tmp_path):
    snap, table = _snapshot(vm, orc, tmp_path)
    k = 1
    _flip(snap / "multi.bin", k * BB + 4096 * 3 + 1)
    dst = tmp_path / "dst"
    dst.mkdir()
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, dst, None, tmp_path / "out.vmig", flags=vm.F_DIRECT_IO),
                    f"multi.bin block {k} ")
    assert not (tmp_path / "out.vmig").exists()


# ------------------------------------------------------------------------------------------ hand-off
def test_rollback_from_a_corrupted_snapshot_raises(vm, orc, shm_tmp):
    ho = _handoff(vm)
    up2, up3 = shm_tmp / "upper_2", shm_tmp / "upper_3"
    up2.mkdir(), up3.mkdir()
    for i in range(3):
        (up2 / f"g{i}.bin").write_bytes(orc.splitmix_bytes(300 + i, 9 * MiB + i).tobytes())
    vm.set_resolver(container_upperdir=lambda n: str({"rs-2": up2, "rs-3": up3}[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersion("rs-2")
        data, table = ho.snapshotPaths("rs-2")
        assert table.exists() and orc.compare_trees(up2, data) == []
        _flip(data / "g1.bin", 5 * MiB)
        with pytest.raises(vm.VmigError) as ei:
            ho.RollbackFromSnapshot("rs-2", "rs-3")
        assert ei.value.code == vm.VMIG_ECORRUPT and "g1.bin block 1 " in str(ei.value)
        assert not ho.snapshotPaths("rs-3")[1].exists()
    finally:
        vm.set_resolver(None, None); ho.set_merges_root(None)


# ------------------------------------------------------------------------------------------ bench scale
def _free_bytes(p) -> int:
    st = os.statvfs(p)
    avail = [st.f_bavail * st.f_frsize]
    for line in Path("/proc/meminfo").read_text().splitlines():
        if line.startswith("MemAvailable:"):
            avail.append(int(line.split()[1]) * 1024)
    return min(avail)


def test_one_flipped_block_among_2560_at_bench_scale(vm, orc, shm_tmp):
    n_files, fbytes = 10, 1 << 30
    if _free_bytes(shm_tmp) < 2.5 * n_files * fbytes:
        pytest.skip("needs ~25 GiB of tmpfs for a 10 x 1 GiB snapshot and its restore")
    snap = shm_tmp / "snap"
    snap.mkdir()
    vm.datagen_files(snap, 0x5EED, n_files, fbytes)
    table = shm_tmp / "snap.vmig"
    vm.hash_tree(snap, table)
    assert vm.table_info(table)["n_blocks"] == 2560
    f, k = "f00007.bin", 123
    old = _flip(snap / f, k * BB + 999)
    dst = shm_tmp / "dst"
    dst.mkdir()
    _expect_corrupt(vm, lambda: vm.restore_tree(snap, table, dst, None, shm_tmp / "out.vmig"), f"{f} block {k} ")
    assert not (shm_tmp / "out.vmig").exists()
    shutil.rmtree(dst)
    with open(snap / f, "r+b") as fh:                          # repaired: the same snapshot restores cleanly
        fh.seek(k * BB + 999)
        fh.write(old)
    dst.mkdir()
    st = vm.restore_tree(snap, table, dst, None, shm_tmp / "out.vmig", flags=vm.F_VERIFY)
    assert st["blocks_total"] == 2560 and st["bytes_written"] == n_files * fbytes
    assert (vm.table_hashes(shm_tmp / "out.vmig") == vm.table_hashes(table)).all()
    for i in range(n_files):
        a, b = snap / f"f{i:05d}.bin", dst / f"f{i:05d}.bin"
        with open(a, "rb") as fa, open(b, "rb") as fb:
            while True:
                x, y = fa.read(64 * MiB), fb.read(64 * MiB)
                assert x == y, a.name
                if not x:
                    break
