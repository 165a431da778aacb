"""vmig_restore_paths on the GPU (-m gpu): chosen entries of a snapshot, each block checked against the snapshot's table.

The result must equal the reference's tar pipe restricted to the same members, run on an identical destination; the cost
must follow the selection; damage inside the selection fails the call before a bad block lands, damage outside it does
not matter; nothing in the destination outside the selection and its parent chains is touched, and no destination
symlink is followed."""
import os
import shutil
import subprocess
import threading
import time
from pathlib import Path

import pytest

from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB = 4 * MiB
T0 = 1_500_000_000_000_000_000


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _snapshot(vm, orc, base: Path, name: str = "snap"):
    """The rich tree plus a multi-block file, copied by the engine into base/<name> with its block table."""
    src, snap = base / f"{name}_src", base / name
    src.mkdir(), snap.mkdir()
    make_rich_tree(src, orc)
    (src / "multi.bin").write_bytes(orc.splitmix_bytes(77, 3 * BB + 4097).tobytes())
    vm.migrate_tree(src, snap, None, base / f"{name}.vmig", flags=vm.F_VERIFY)
    return snap, base / f"{name}.vmig"


def _flip(path: Path, off: int) -> int:
    """XOR one byte of the file in place; returns the byte's new value."""
    with open(path, "r+b") as f:
        f.seek(off)
        new = f.read(1)[0] ^ 0x5A
        f.seek(off)
        f.write(bytes([new]))
    return new


def _state(root: Path) -> dict:
    """Every entry under root with its kind, owner, content and mtime: what 'untouched' means."""
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for n in [""] + dirnames + filenames:
            p = os.path.join(dirpath, n) if n else dirpath
            st = os.lstat(p)
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[os.path.relpath(p, root)] = (st.st_mode, st.st_uid, st.st_gid, st.st_mtime_ns, body)
    return out


def _prepopulated(dst: Path) -> Path:
    """A destination whose parents exist, with entries in and out of the selection."""
    (dst / "sub" / "deep").mkdir(parents=True)
    (dst / "keep_dir").mkdir()
    (dst / "stale.bin").write_bytes(b"s" * 5000)
    (dst / "sub" / "small.txt").write_bytes(b"old")
    (dst / "sub" / "extra_in_sub").write_bytes(b"extra")
    (dst / "multi.bin").write_bytes(b"m" * 10000)
    (dst / "keep_dir" / "k").write_bytes(b"k")
    (dst / "big.bin").write_bytes(b"b" * 100)
    os.symlink("stale.bin", dst / "lnk_old")
    for dirpath, dirnames, filenames in os.walk(dst, topdown=False):      # children before their directory
        for n in dirnames + filenames:
            os.utime(os.path.join(dirpath, n), ns=(T0, T0), follow_symlinks=False)
    os.utime(dst, ns=(T0, T0))
    return dst


def _under(rel: str, paths) -> bool:
    return any(rel == p or rel.startswith(p + "/") for p in paths)


def _expect(vm, code, call, *needles):
    with pytest.raises(vm.VmigError) as ei:
        call()
    assert ei.value.code == code, ei.value
    for n in needles:
        assert n in str(ei.value), ei.value
    return ei.value


# ------------------------------------------------------------------------------------------ 1. parity with tar
@pytest.mark.parametrize("lanes", [1, 2])
def test_equals_the_tar_pipe_restricted_to_members(vm, orc, shm_tmp, lanes):
    snap, table = _snapshot(vm, orc, shm_tmp)
    members = ["sub", "big.bin", "lnk", "fifo"]
    dst, ref = _prepopulated(shm_tmp / "dst"), _prepopulated(shm_tmp / "ref")
    before = _state(dst)
    st = vm.restore_paths(snap, table, dst, members, lanes_per_gpu=lanes)
    subprocess.run(f"(cd {snap}; tar c -- {' '.join(members)}) | (cd {ref}; tar x)", shell=True, check=True)
    assert orc.compare_trees(ref, dst, ignore_root_mtime=True) == []
    after = _state(dst)
    for rel, s in before.items():
        if rel != "." and not _under(rel, members):
            assert after[rel] == s, rel
    assert (st["files"], st["hardlinks"], st["symlinks"], st["specials"]) == (4, 1, 2, 1)


# ------------------------------------------------------------------------------------------ 2. cost
def test_cost_follows_the_selection(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    chosen = ["big.bin", "sub/small.txt"]       # both have a hard-link partner outside the selection: files of their own
    size = sum(os.path.getsize(snap / p) for p in chosen)
    blocks = sum(-(-os.path.getsize(snap / p) // BB) for p in chosen)
    for flags, reads in ((0, 1), (vm.F_VERIFY, 2)):
        dst = shm_tmp / f"dst{flags}"
        dst.mkdir()
        with vm.Ctl() as ctl:
            st = vm.restore_paths(snap, table, dst, chosen, flags=flags, ctl=ctl)
            p = ctl.progress()
        assert st["bytes_total"] == size and st["blocks_total"] == blocks and st["files"] == 2
        assert st["bytes_h2d"] == reads * size and st["bytes_written"] == size
        assert p["bytes_total"] == size and p["blocks_total"] == blocks and p["phase_name"] == "DONE"
        assert sorted(os.listdir(dst)) == ["big.bin", "sub"] and os.listdir(dst / "sub") == ["small.txt"]
        assert os.stat(dst / "big.bin").st_nlink == 1


# ------------------------------------------------------------------------------------------ 3. damaged blocks
def test_damaged_block_inside_the_selection_is_never_written(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    off = BB + 10
    bad = _flip(snap / "multi.bin", off)
    dst = shm_tmp / "dst"
    dst.mkdir()
    _expect(vm, vm.VMIG_ECORRUPT, lambda: vm.restore_paths(snap, table, dst, ["multi.bin", "exact.bin"]), "multi.bin block 1 ")
    p = dst / "multi.bin"
    if p.exists() and p.stat().st_size > off:
        with open(p, "rb") as f:
            f.seek(off)
            assert f.read(1)[0] != bad


def test_damage_outside_the_selection_does_not_matter(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    _flip(snap / "multi.bin", 5)
    _flip(snap / ".hidden_dir" / "inner", 5)
    dst = shm_tmp / "dst"
    dst.mkdir()
    vm.restore_paths(snap, table, dst, ["big.bin", "sub"], flags=vm.F_VERIFY)
    assert (dst / "big.bin").read_bytes() == (snap / "big.bin").read_bytes()
    assert (dst / "sub" / "deep" / "tiny").read_bytes() == b"abc"


# ------------------------------------------------------------------------------------------ 4. missing / extra / resized
@pytest.mark.parametrize("change,chosen,needle", [
    ("missing", ["sub"], "sub/small.txt is in the block table but not in the snapshot (missing)"),
    ("extra", ["sub"], "sub/new.txt is in the snapshot but not in its block table (extra)"),
    ("resized", ["sub"], "sub/deep/tiny is 4 bytes in the snapshot, 3 in its block table (resized)"),
    ("chosen_missing", ["exact.bin", "big.bin"], "exact.bin is in the block table but not in the snapshot (missing)"),
])
def test_table_mismatch_inside_the_selection(vm, orc, shm_tmp, change, chosen, needle):
    snap, table = _snapshot(vm, orc, shm_tmp)
    {"missing": lambda: (snap / "sub" / "small.txt").unlink(),
     "extra": lambda: (snap / "sub" / "new.txt").write_bytes(b"new"),
     "resized": lambda: (snap / "sub" / "deep" / "tiny").write_bytes(b"abcd"),
     "chosen_missing": lambda: (snap / "exact.bin").unlink()}[change]()
    dst = _prepopulated(shm_tmp / "dst")
    before = _state(dst)
    _expect(vm, vm.VMIG_ECORRUPT, lambda: vm.restore_paths(snap, table, dst, chosen, flags=vm.F_PRUNE), needle)
    assert _state(dst) == before
    # outside the selection the same damage does not matter
    vm.restore_paths(snap, table, dst, ["multi.bin", "lnk"])
    assert (dst / "multi.bin").read_bytes() == (snap / "multi.bin").read_bytes()


def test_path_not_in_the_snapshot(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst = _prepopulated(shm_tmp / "dst")
    before = _state(dst)
    _expect(vm, vm.VMIG_EINVAL, lambda: vm.restore_paths(snap, table, dst, ["big.bin", "sub/nothere"]),
            "sub/nothere is not in the snapshot")
    _expect(vm, vm.VMIG_EINVAL, lambda: vm.restore_paths(snap, table, dst, ["lnk/x"]), "lnk/x is not in the snapshot")
    assert _state(dst) == before


# ------------------------------------------------------------------------------------------ 5. destination symlinks
def test_destination_symlinks_are_replaced_never_followed(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    outside = shm_tmp / "outside"
    (outside / "deep").mkdir(parents=True)
    (outside / "deep" / "tiny").write_bytes(b"outside")
    (outside / "file.bin").write_bytes(b"outside file")
    dst = shm_tmp / "dst"
    dst.mkdir()
    os.symlink(outside, dst / "sub")
    os.symlink(outside / "file.bin", dst / "big.bin")
    before = _state(outside)
    vm.restore_paths(snap, table, dst, ["sub/deep/tiny", "big.bin"], flags=vm.F_VERIFY)
    assert _state(outside) == before
    assert not (dst / "sub").is_symlink() and (dst / "sub").is_dir()
    assert (dst / "sub" / "deep" / "tiny").read_bytes() == b"abc"
    assert not (dst / "big.bin").is_symlink() and (dst / "big.bin").read_bytes() == (snap / "big.bin").read_bytes()


# ------------------------------------------------------------------------------------------ 6. missing parents
def test_missing_parents_take_the_snapshots_metadata(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst = shm_tmp / "dst"
    dst.mkdir()
    (dst / "keep").mkdir()
    os.chmod(dst / "keep", 0o750)
    vm.restore_paths(snap, table, dst, ["sub/deep/tiny"])
    for rel in ("sub", "sub/deep"):
        s, d = os.lstat(snap / rel), os.lstat(dst / rel)
        assert d.st_mode == s.st_mode, rel
        assert d.st_mtime_ns // 10**9 == s.st_mtime_ns // 10**9, rel
        if os.geteuid() == 0:
            assert (d.st_uid, d.st_gid) == (s.st_uid, s.st_gid), rel
    if os.geteuid() == 0:
        assert (os.lstat(dst / "sub").st_uid, os.lstat(dst / "sub").st_gid) == (1234, 4321)
    assert os.lstat(dst / "sub" / "deep").st_mode & 0o7777 == 0o711
    assert sorted(os.listdir(dst)) == ["keep", "sub"] and os.listdir(dst / "sub") == ["deep"]
    assert os.lstat(dst / "keep").st_mode & 0o7777 == 0o750


# ------------------------------------------------------------------------------------------ 7. hard links
def test_hard_links_inside_the_selection_only(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    both, alone = shm_tmp / "both", shm_tmp / "alone"
    both.mkdir(), alone.mkdir()
    st = vm.restore_paths(snap, table, both, ["big.bin", "sub/hard1"], flags=vm.F_VERIFY)
    a, b = os.lstat(both / "big.bin"), os.lstat(both / "sub" / "hard1")
    assert a.st_ino == b.st_ino and a.st_nlink == 2 and st["hardlinks"] == 1
    vm.restore_paths(snap, table, alone, ["sub/hard1"])
    h = os.lstat(alone / "sub" / "hard1")
    assert h.st_nlink == 1 and (alone / "sub" / "hard1").read_bytes() == (snap / "big.bin").read_bytes()


# ------------------------------------------------------------------------------------------ 8. prune
def test_prune_stays_beneath_the_chosen_directories(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst = _prepopulated(shm_tmp / "dst")
    (dst / "sub" / "deep" / "extra_dir").mkdir()
    (dst / "sub" / "deep" / "extra_dir" / "x").write_bytes(b"x")
    (dst / "sub" / "deep" / "extra_file").write_bytes(b"y")
    os.symlink(dst / "keep_dir", dst / "sub" / "deep" / "extra_link")
    st = vm.restore_paths(snap, table, dst, ["sub/deep"], flags=vm.F_PRUNE)
    assert st["pruned"] == 4
    assert sorted(os.listdir(dst / "sub" / "deep")) == ["tiny"]
    assert (dst / "sub" / "extra_in_sub").read_bytes() == b"extra"      # a sibling of the chosen directory
    assert (dst / "stale.bin").exists() and (dst / "keep_dir" / "k").exists() and os.path.islink(dst / "lnk_old")
    dst2 = _prepopulated(shm_tmp / "dst2")
    (dst2 / "sub" / "gone").write_bytes(b"g")
    st = vm.restore_paths(snap, table, dst2, ["sub", "big.bin", "a_hard2"], flags=vm.F_VERIFY | vm.F_PRUNE)
    assert st["pruned"] == 2 and not (dst2 / "sub" / "extra_in_sub").exists() and (dst2 / "stale.bin").exists()
    assert orc.compare_trees(snap / "sub", dst2 / "sub") == []


# ------------------------------------------------------------------------------------------ 9. prior table
def test_prior_table_writes_only_changed_blocks(vm, orc, shm_tmp):
    src = shm_tmp / "src"
    src.mkdir()
    make_rich_tree(src, orc)
    body = bytearray(orc.splitmix_bytes(77, 3 * BB + 4097).tobytes())
    (src / "multi.bin").write_bytes(body)
    snap_a, snap_b = shm_tmp / "A", shm_tmp / "B"
    snap_a.mkdir(), snap_b.mkdir()
    vm.migrate_tree(src, snap_a, None, shm_tmp / "A.vmig")
    body[BB + 7] ^= 0xFF                          # version B differs from A in one block of multi.bin
    st_m = os.stat(src / "multi.bin")
    (src / "multi.bin").write_bytes(body)
    os.utime(src / "multi.bin", ns=(st_m.st_atime_ns, st_m.st_mtime_ns))
    vm.migrate_tree(src, snap_b, None, shm_tmp / "B.vmig")
    dst = shm_tmp / "dst"
    dst.mkdir()
    vm.restore_tree(snap_a, shm_tmp / "A.vmig", dst, None, shm_tmp / "dst.vmig")
    ex = os.lstat(dst / "exact.bin")
    st = vm.restore_paths(snap_b, shm_tmp / "B.vmig", dst, ["multi.bin", "exact.bin"], shm_tmp / "dst.vmig")
    assert st["bytes_written"] == BB and st["files_untrusted"] == 0
    assert (dst / "multi.bin").read_bytes() == bytes(body)
    ex2 = os.lstat(dst / "exact.bin")
    assert (ex2.st_ino, ex2.st_ctime_ns) == (ex.st_ino, ex.st_ctime_ns)


# ------------------------------------------------------------------------------------------ 10. control
def test_control(vm, orc, shm_tmp):
    snap, table = _snapshot(vm, orc, shm_tmp)
    dst = _prepopulated(shm_tmp / "dst")
    before = _state(dst)
    with vm.Ctl() as ctl:
        ctl.cancel()
        _expect(vm, vm.VMIG_ECANCELED, lambda: vm.restore_paths(snap, table, dst, ["sub", "big.bin"], ctl=ctl))
    assert _state(dst) == before

    big = shm_tmp / "bigsnap"
    (big / "d").mkdir(parents=True)
    vm.datagen_files(big / "d", 5, 8, 128 * MiB)
    vm.hash_tree(big, shm_tmp / "big.vmig")
    out = shm_tmp / "out"
    out.mkdir()
    with vm.Ctl() as ctl:
        res = {}

        def cancel_in_data():
            t_end = time.monotonic() + 60
            while time.monotonic() < t_end:
                p = ctl.progress()
                if p["phase_name"] == "DATA" and p["bytes_hashed"] > 0:
                    ctl.cancel()
                    return
                time.sleep(0.0005)
        t = threading.Thread(target=cancel_in_data)
        t.start()
        try:
            vm.restore_paths(big, shm_tmp / "big.vmig", out, ["d"], ctl=ctl)
        except vm.VmigError as e:
            res["err"] = e
        t.join()
        assert "err" in res and res["err"].code == vm.VMIG_ECANCELED, res
        assert "cancelled in phase DATA" in str(res["err"])
        assert ctl.progress()["running"] == 0          # detached: it can be read and closed; a cancel on it is final
    with vm.Ctl() as ctl:
        st = vm.restore_paths(big, shm_tmp / "big.vmig", out, ["d"], flags=vm.F_VERIFY, ctl=ctl)
        p = ctl.progress()
        assert p["phase_name"] == "DONE" and p["running"] == 0
        assert (p["bytes_total"], p["blocks_total"]) == (st["bytes_total"], st["blocks_total"]) == (8 * 128 * MiB, 8 * 32)
        assert p["bytes_hashed"] == st["bytes_total"] and p["bytes_verified"] == st["bytes_total"]
    assert orc.compare_trees(big / "d", out / "d") == []


# ------------------------------------------------------------------------------------------ 11. the hand-off mirror
def test_restore_paths_from_snapshot_mirror(vm, orc, shm_tmp):
    import importlib
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {n: shm_tmp / f"upper_{n}" for n in ("rs-1", "rs-2", "rs-3")}
    for p in ups.values():
        p.mkdir()
    make_rich_tree(ups["rs-1"], orc)
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersion("rs-1")
        # the tenant's layer moves on: rs-2 is the running container, rs-3 its Patch successor
        shutil.rmtree(ups["rs-2"])
        subprocess.run(f"(cd {ups['rs-1']}; tar c .) | (cd {shm_tmp}; mkdir upper_rs-2; cd upper_rs-2; tar x)", shell=True, check=True)
        (ups["rs-2"] / "big.bin").write_bytes(b"overwritten")
        shutil.rmtree(ups["rs-2"] / "sub")
        (ups["rs-2"] / "new_since.txt").write_bytes(b"keep me")
        (ups["rs-2"] / "exact.bin").write_bytes(b"changed since")
        ho.HandoffCopy("rs-2", "rs-3", pause=lambda n: None, resume=lambda n: None)
        _, seed = ho.snapshotPaths("rs-3")
        st = ho.RestorePathsFromSnapshot("rs-1", "rs-3", ["sub", "big.bin"], seed)
        want = shm_tmp / "want"
        want.mkdir()
        subprocess.run(f"(cd {ups['rs-2']}; tar c .) | (cd {want}; tar x)", shell=True, check=True)
        (want / "big.bin").unlink()
        data, _ = ho.snapshotPaths("rs-1")
        subprocess.run(f"(cd {data}; tar c -- sub big.bin) | (cd {want}; tar x)", shell=True, check=True)
        assert orc.compare_trees(want, ups["rs-3"], ignore_root_mtime=True) == []
        assert st["files"] == 4 and (ups["rs-3"] / "new_since.txt").read_bytes() == b"keep me"
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
