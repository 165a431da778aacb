"""vmig_snapshot_tree on the GPU (-m gpu): an incremental snapshot finds unchanged content in its base by block hash,
wherever the base holds it -- a file renamed, moved to another directory, copied, swapped with another, or shifted by
whole blocks -- not only at the same path and offset.

Each case builds v1 with snapshot_tree and then v2 against it.  v2 must equal the reference's tar copy of the source,
carry the oracle's block table and restore exactly; v1 must not change."""
import collections
import os
import shutil
import time
from pathlib import Path

import pytest

from test_cancel import _cancelled, _run

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB = 4 * MiB


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _snap(vm, src: Path, dst: Path, base: Path = None, flags=None, **kw):
    """Snapshot src into the new directory dst, table next to it as <dst>.vmig; base's table is <base>.vmig."""
    dst.mkdir()
    out = dst.with_name(dst.name + ".vmig")
    bt = None if base is None else base.with_name(base.name + ".vmig")
    return vm.snapshot_tree(src, dst, base, bt, out, flags=vm.F_VERIFY if flags is None else flags, **kw), out


def _state(root: Path) -> dict:
    """Every entry under root with its kind, content and mtime: what 'untouched' means."""
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for n in [""] + dirnames + filenames:
            p = os.path.join(dirpath, n) if n else dirpath
            st = os.lstat(p)
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[os.path.relpath(p, root)] = (st.st_mode, st.st_mtime_ns, body)
    return out


def _tree(orc, root) -> dict:
    """The oracle's manifest of root, with hard-link groups as seen INSIDE the tree: a file whose only other links are
    in another snapshot is a plain file here."""
    m = orc.tree_manifest(root)
    size = collections.Counter(r["hardlink_to"] for r in m.values() if "hardlink_to" in r)
    for r in m.values():
        if "hardlink_to" in r and size[r["hardlink_to"]] < 2:
            del r["hardlink_to"]
    return m


def _check(vm, orc, src: Path, snap: Path, table: Path):
    """snap equals the tar copy of src, its table the oracle's, and it restores to that tar copy."""
    ref = snap.with_name("ref_" + snap.name)
    ref.mkdir()
    orc.ref_copy(src, ref)
    ta, tb = _tree(orc, ref), _tree(orc, snap)
    diffs = [k for k in sorted(set(ta) | set(tb)) if ta.get(k) != tb.get(k)]
    assert not diffs, [(k, ta.get(k), tb.get(k)) for k in diffs[:5]]
    _, want = orc.block_table_of_tree(src)
    assert (vm.table_hashes(table) == want).all()
    dst = snap.with_name("restore_" + snap.name)
    dst.mkdir()
    vm.restore_tree(snap, table, dst, None, None, flags=vm.F_VERIFY)
    assert orc.compare_trees(ref, dst) == []
    shutil.rmtree(dst)
    shutil.rmtree(ref)


def _ino(p: Path) -> int:
    return os.lstat(p).st_ino


def _put(orc, p: Path, seed: int, size: int):
    p.parent.mkdir(parents=True, exist_ok=True)
    p.write_bytes(orc.splitmix_bytes(seed, size).tobytes())


def _v1(vm, orc, root: Path, files: dict, flags=None):
    """src with files {rel: (seed, size)}, snapshot v1 of it; returns src, v1, v2 (not yet made), v1's state."""
    src, v1 = root / "src", root / "v1"
    for rel, (seed, size) in files.items():
        _put(orc, src / rel, seed, size)
    _snap(vm, src, v1, flags=flags)
    return src, v1, root / "v2", _state(v1)


def _v2(vm, orc, src, v1, v2, before, flags=None, **kw):
    st, t2 = _snap(vm, src, v2, v1, flags=flags, **kw)
    _check(vm, orc, src, v2, t2)
    assert _state(v1) == before
    return st


# ------------------------------------------------------------------------------------------ moved, unchanged
def test_renamed_into_a_new_directory_is_linked(vm, orc, shm_tmp):
    size = 3 * BB + 4097                                   # a short last block
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"a/big.bin": (1, size), "a/keep.bin": (2, BB + 7)})
    (src / "b").mkdir()
    os.rename(src / "a" / "big.bin", src / "b" / "moved.bin")
    st = _v2(vm, orc, src, v1, v2, before)
    assert _ino(v2 / "b" / "moved.bin") == _ino(v1 / "a" / "big.bin")
    assert st["bytes_written"] == 0 and st["bytes_d2h"] == 0, st
    assert st["files_linked"] == 2 and st["bytes_linked"] == size + BB + 7 and st["files_backfilled"] == 0, st
    assert st["blocks_skipped"] == st["blocks_total"] and st["files_base_untrusted"] == 0, st


@pytest.mark.parametrize("lanes", [1, 3])
def test_every_file_moved(vm, orc, shm_tmp, lanes):
    """No source path has a same-path base record: the call still runs in skip mode and streams nothing back."""
    files = {f"old/f{i}.bin": (10 + i, (i + 1) * BB + 333 * i) for i in range(6)}
    src, v1, v2, before = _v1(vm, orc, shm_tmp, files)
    os.rename(src / "old", src / "new")
    st = _v2(vm, orc, src, v1, v2, before, lanes_per_gpu=lanes)
    for i in range(6):
        assert _ino(v2 / "new" / f"f{i}.bin") == _ino(v1 / "old" / f"f{i}.bin"), i
    assert st["bytes_written"] == 0 and st["bytes_d2h"] == 0 and st["files_linked"] == 6, st
    assert st["lanes_used"] >= lanes, st


def test_swapped_pair_links_each_to_the_other(vm, orc, shm_tmp):
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"a": (20, 2 * BB + 1), "b": (21, BB + 5)})
    os.rename(src / "a", src / "tmp")
    os.rename(src / "b", src / "a")
    os.rename(src / "tmp", src / "b")
    st = _v2(vm, orc, src, v1, v2, before)
    assert _ino(v2 / "a") == _ino(v1 / "b") and _ino(v2 / "b") == _ino(v1 / "a")
    assert st["files_linked"] == 2 and st["bytes_written"] == 0 and st["bytes_d2h"] == 0, st


# ------------------------------------------------------------------------------------------ copies
def test_copy_with_a_new_mtime_is_backfilled_from_the_original(vm, orc, shm_tmp):
    size = 2 * BB + 999
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"ckpt_latest/model.pt": (30, size)})
    time.sleep(1.1)                                        # the copy's mtime differs in whole seconds too
    (src / "best").mkdir()
    shutil.copyfile(src / "ckpt_latest" / "model.pt", src / "best" / "model.pt")
    st = _v2(vm, orc, src, v1, v2, before)
    assert _ino(v2 / "ckpt_latest" / "model.pt") == _ino(v1 / "ckpt_latest" / "model.pt")
    assert _ino(v2 / "best" / "model.pt") != _ino(v1 / "ckpt_latest" / "model.pt")
    assert st["files_linked"] == 1 and st["files_backfilled"] == 1 and st["bytes_backfilled"] == size, st
    assert st["bytes_written"] == 0 and st["bytes_d2h"] == 0, st


def test_two_new_paths_with_one_base_files_content(vm, orc, shm_tmp):
    size = 3 * BB
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"orig.bin": (40, size)})
    o = os.lstat(src / "orig.bin")
    for n in ("p1.bin", "p2.bin"):
        shutil.copyfile(src / "orig.bin", src / n)
        os.utime(src / n, ns=(o.st_atime_ns, o.st_mtime_ns))
    os.unlink(src / "orig.bin")
    st = _v2(vm, orc, src, v1, v2, before)
    assert sorted([_ino(v2 / "p1.bin") == _ino(v1 / "orig.bin"), _ino(v2 / "p2.bin") == _ino(v1 / "orig.bin")]) == [False, True]
    assert st["files_linked"] == 1 and st["files_backfilled"] == 1 and st["bytes_backfilled"] == size, st
    assert st["bytes_written"] == 0, st


def test_base_inode_linked_and_backfilled_in_one_call(vm, orc, shm_tmp):
    """Each x_i keeps its path (a link to v1's file), its copy y_i takes every byte from that same base inode: whichever
    finishes first, the other sees the ctime this call's own link left, which is not a change of the base."""
    n, size = 8, BB + 4096 * 3
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {f"x{i}.bin": (50 + i, size) for i in range(n)})
    time.sleep(1.1)
    for i in range(n):
        shutil.copyfile(src / f"x{i}.bin", src / f"y{i}.bin")
    st = _v2(vm, orc, src, v1, v2, before, lanes_per_gpu=3)
    for i in range(n):
        assert _ino(v2 / f"x{i}.bin") == _ino(v1 / f"x{i}.bin")
    assert st["files_linked"] == n and st["files_backfilled"] == n and st["bytes_written"] == 0, st


# ------------------------------------------------------------------------------------------ partly changed
def test_renamed_file_with_one_changed_block_writes_only_that_block(vm, orc, shm_tmp):
    size = 4 * BB + 10
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"run1/data.bin": (60, size)})
    os.rename(src / "run1", src / "run2")
    with open(src / "run2" / "data.bin", "r+b") as f:
        f.seek(2 * BB + 5)
        f.write(b"\xa5" * 100)
    st = _v2(vm, orc, src, v1, v2, before)
    assert st["bytes_written"] == BB and st["bytes_d2h"] == BB, st
    assert st["files_linked"] == 0 and st["files_backfilled"] == 1 and st["bytes_backfilled"] == size - BB, st


def test_first_block_cut_off_reuses_the_old_blocks_at_lower_offsets(vm, orc, shm_tmp):
    size = 5 * BB + 777
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {"log.bin": (70, size)})
    body = (src / "log.bin").read_bytes()
    (src / "log.bin").write_bytes(body[BB:])
    st = _v2(vm, orc, src, v1, v2, before)
    assert st["bytes_written"] == 0 and st["bytes_d2h"] == 0, st
    assert st["files_backfilled"] == 1 and st["bytes_backfilled"] == size - BB and st["blocks_skipped"] == 5, st


# ------------------------------------------------------------------------------------------ untrusted base
def test_moved_files_base_copy_rewritten_out_of_band_is_not_reused(vm, orc, shm_tmp):
    size = 2 * BB + 3
    src, v1, v2, _ = _v1(vm, orc, shm_tmp, {"m.bin": (80, size), "k.bin": (81, BB)})
    time.sleep(0.05)
    p = v1 / "m.bin"
    old = os.lstat(p)
    p.write_bytes(orc.splitmix_bytes(99, size).tobytes())          # same inode and size, other bytes ...
    os.utime(p, ns=(old.st_atime_ns, old.st_mtime_ns))             # ... and the mtime put back
    before = _state(v1)
    os.rename(src / "m.bin", src / "moved.bin")
    st = _v2(vm, orc, src, v1, v2, before)
    assert _ino(v2 / "moved.bin") != _ino(p)
    assert st["bytes_written"] == size and st["files_linked"] == 1 and st["files_backfilled"] == 0, st


def test_base_table_written_for_another_directory_reuses_nothing(vm, orc, shm_tmp):
    src, v1, v2, before = _v1(vm, orc, shm_tmp, {f"f{i}.bin": (90 + i, BB + 1000 * i) for i in range(3)})
    layer = shm_tmp / "layer"
    layer.mkdir()
    vm.migrate_tree(src, layer, None, shm_tmp / "v1.vmig")          # v1.vmig now speaks for layer/, not for v1/
    for i in range(3):
        os.rename(src / f"f{i}.bin", src / f"g{i}.bin")
    st = _v2(vm, orc, src, v1, v2, before)
    assert st["files_linked"] == 0 and st["files_backfilled"] == 0 and st["blocks_skipped"] == 0, st
    assert st["bytes_written"] == st["bytes_total"], st


# ------------------------------------------------------------------------------------------ O_DIRECT, verify
def test_direct_io_reuse_with_a_partial_last_sector(vm, orc, tmp_path):
    """A non-tmpfs tree with VMIG_F_DIRECT_IO and VMIG_F_VERIFY: moved, copied and shifted content backfilled through
    the O_DIRECT destination, last blocks ending inside a sector."""
    f = vm.F_VERIFY | vm.F_DIRECT_IO
    size = 2 * BB + 1000
    src, v1, v2, before = _v1(vm, orc, tmp_path, {"d.bin": (100, size), "s.bin": (101, 3 * BB + 512)}, flags=f)
    os.rename(src / "d.bin", src / "moved.bin")
    time.sleep(1.1)
    shutil.copyfile(src / "moved.bin", src / "copy.bin")
    body = (src / "s.bin").read_bytes()
    (src / "s.bin").write_bytes(body[BB:])
    st = _v2(vm, orc, src, v1, v2, before, flags=f)
    assert st["bytes_written"] == 0 and st["files_linked"] == 1, st
    assert st["files_backfilled"] == 2 and st["bytes_backfilled"] == size + 2 * BB + 512, st
    assert (v2 / "copy.bin").read_bytes() == (src / "copy.bin").read_bytes()


# ------------------------------------------------------------------------------------------ cancel
def test_cancel_during_a_cross_path_backfill(vm, orc, shm_tmp):
    src, v1 = shm_tmp / "src", shm_tmp / "v1"
    (src / "a").mkdir(parents=True)
    vm.datagen_files(src / "a", 5, 1, 1024 * MiB)
    v1.mkdir()
    t1 = shm_tmp / "v1.vmig"
    vm.snapshot_tree(src, v1, None, None, t1)
    os.rename(src / "a", src / "b")
    with open(src / "b" / "f00000.bin", "r+b") as f:   # one changed block: the other 255 come from v1/a/f00000.bin
        f.seek(100 * BB)
        f.write(b"\x5a" * 4096)
    before, table_before = _state(v1), t1.read_bytes()
    backfill = lambda p: p["phase_name"] == "DATA" and p["blocks_total"] and p["blocks_hashed"] == p["blocks_total"]  # noqa: E731
    out = shm_tmp / "v2.vmig"
    (shm_tmp / "v2").mkdir()
    with vm.Ctl() as ctl:
        res, lat, _ = _run(lambda: vm.snapshot_tree(src, shm_tmp / "v2", v1, t1, out, flags=vm.F_VERIFY, ctl=ctl), ctl, backfill)
        _cancelled(vm, res, lat)
    assert not out.exists() and not [n for n in os.listdir(shm_tmp) if n.startswith("v2.vmig.tmp")]
    assert _state(v1) == before and t1.read_bytes() == table_before
    st = _v2(vm, orc, src, v1, shm_tmp / "v3", before)
    assert st["files_backfilled"] == 1 and st["bytes_written"] == BB, st


# ------------------------------------------------------------------------------------------ hand-off
def test_handoff_incremental_snapshot_after_a_directory_rename(vm, orc, shm_tmp):
    import importlib
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {f"rs-{i}": shm_tmp / f"upper_{i}" for i in (2, 3)}
    for p in ups.values():
        p.mkdir()
    for i in range(3):
        _put(orc, ups["rs-2"] / "ckpt_latest" / f"g{i}.bin", 300 + i, 9 * MiB + i)
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersionIncremental("rs-2")
        orc.ref_copy(ups["rs-2"], ups["rs-3"])
        os.rename(ups["rs-3"] / "ckpt_latest", ups["rs-3"] / "ckpt_1200")
        assert ho.baseVersion("rs-3") == "rs-2"
        st3 = ho.SnapshotVersionIncremental("rs-3")
        assert st3["files_linked"] == 3 and st3["bytes_written"] == 0 and st3["bytes_d2h"] == 0, st3
        for i in range(3):
            assert (_ino(ho.versionDir("rs-3") / "diff" / "ckpt_1200" / f"g{i}.bin")
                    == _ino(ho.versionDir("rs-2") / "diff" / "ckpt_latest" / f"g{i}.bin"))
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
