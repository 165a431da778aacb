"""vmig_snapshot_tree on the GPU (-m gpu): incremental version snapshots that share unchanged files (hard links) and
unchanged blocks (copied from the base file on the host) with the previous snapshot.

Every snapshot must equal the reference's tar copy of its source, carry the oracle's block table, and restore exactly
with vmig_restore_tree; the base snapshot must never change, whatever the increment links to it."""
import collections
import os
import shutil
import time
from pathlib import Path

import pytest

from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB = 4 * MiB


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _tree(orc, root) -> dict:
    """The oracle's manifest of root, with hard-link groups as seen INSIDE the tree: a file whose only other links are
    in another snapshot is a plain file here."""
    m = orc.tree_manifest(root)
    size = collections.Counter(r["hardlink_to"] for r in m.values() if "hardlink_to" in r)
    for r in m.values():
        if "hardlink_to" in r and size[r["hardlink_to"]] < 2:
            del r["hardlink_to"]
    return m


def _same(orc, a, b):
    ta, tb = _tree(orc, a), _tree(orc, b)
    diffs = [k for k in sorted(set(ta) | set(tb)) if ta.get(k) != tb.get(k)]
    assert not diffs, [(k, ta.get(k), tb.get(k)) for k in diffs[:5]]


def _snap(vm, src: Path, dst: Path, base: Path = None, flags=None, **kw):
    """Snapshot src into the new directory dst, table next to it as <dst>.vmig; base's table is <base>.vmig."""
    dst.mkdir()
    out = dst.with_name(dst.name + ".vmig")
    bt = None if base is None else base.with_name(base.name + ".vmig")
    st = vm.snapshot_tree(src, dst, base, bt, out, flags=vm.F_VERIFY if flags is None else flags, **kw)
    return st, out


def _check(vm, orc, src: Path, snap: Path, table: Path) -> Path:
    """snap equals the tar copy of src, its table the oracle's, and it restores to that tar copy.  Returns the copy."""
    ref = snap.with_name("ref_" + snap.name)
    ref.mkdir()
    orc.ref_copy(src, ref)
    _same(orc, ref, snap)
    _, want = orc.block_table_of_tree(src)
    assert (vm.table_hashes(table) == want).all()
    _restores(vm, orc, snap, table, ref)
    return ref


def _restores(vm, orc, snap: Path, table: Path, ref: Path):
    dst = snap.with_name("restore_" + snap.name)
    shutil.rmtree(dst, ignore_errors=True)
    dst.mkdir()
    vm.restore_tree(snap, table, dst, None, None, flags=vm.F_VERIFY)
    assert orc.compare_trees(ref, dst) == []
    shutil.rmtree(dst)


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


def _flip(path: Path, off: int):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x5A]))


def _regular(root: Path):
    for dirpath, _, filenames in os.walk(root):
        for n in filenames:
            p = Path(dirpath) / n
            st = os.lstat(p)
            if p.is_file() and not p.is_symlink():
                yield str(p.relative_to(root)), st


# ------------------------------------------------------------------------------------------ unchanged layer
def test_unchanged_layer_links_every_file_without_a_hard_link_partner(vm, orc, shm_tmp):
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    src.mkdir()
    make_rich_tree(src, orc)
    (src / "multi.bin").write_bytes(orc.splitmix_bytes(77, 3 * BB + 4097).tobytes())
    _snap(vm, src, v1)
    st, t2 = _snap(vm, src, v2, v1)
    solo = {rel: s.st_size for rel, s in _regular(src) if s.st_nlink == 1 and s.st_size}
    paired = {rel: s.st_size for rel, s in _regular(src) if s.st_nlink > 1}
    assert len(solo) == 6 and len(paired) == 4
    for rel in solo:
        assert os.lstat(v2 / rel).st_ino == os.lstat(v1 / rel).st_ino, rel
    for rel in paired:                        # the source's hard-link pairs stay pairs of their own
        assert os.lstat(v2 / rel).st_ino != os.lstat(v1 / rel).st_ino, rel
    assert os.lstat(v2 / "big.bin").st_ino == os.lstat(v2 / "sub" / "hard1").st_ino
    assert st["bytes_written"] == 0 and st["bytes_d2h"] == 0, st
    assert st["files_linked"] == 6 and st["bytes_linked"] == sum(solo.values()), st
    # each pair's first path takes all of its blocks from the base file; the second is a link to it
    assert st["files_backfilled"] == 2 and st["bytes_backfilled"] == (src / "big.bin").stat().st_size + 4097, st
    assert st["files_base_untrusted"] == 0, st
    _check(vm, orc, src, v2, t2)


# ------------------------------------------------------------------------------------------ mixed change
@pytest.mark.parametrize("lanes", [1, 3])
def test_mixed_change(vm, orc, shm_tmp, lanes):
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    src.mkdir()
    sizes = {"same.bin": 2 * BB + 5, "flip.bin": 3 * BB + 4097, "grow.bin": BB + 100, "cut.bin": 2 * BB + 10,
             "mode.bin": BB + 1, "gone.bin": 5000}
    for i, (n, size) in enumerate(sizes.items()):
        (src / n).write_bytes(orc.splitmix_bytes(40 + i, size).tobytes())
    _, t1 = _snap(vm, src, v1)
    ref1 = v1.with_name("ref1")
    ref1.mkdir()
    orc.ref_copy(src, ref1)
    before = _state(v1)

    _flip(src / "flip.bin", BB + 17)
    with open(src / "grow.bin", "ab") as f:
        f.write(b"g" * MiB)
    os.truncate(src / "cut.bin", BB + 5)
    os.chmod(src / "mode.bin", 0o600)
    (src / "new.bin").write_bytes(orc.splitmix_bytes(50, BB + 3).tobytes())
    os.unlink(src / "gone.bin")
    st, t2 = _snap(vm, src, v2, v1, lanes_per_gpu=lanes)

    assert os.lstat(v2 / "same.bin").st_ino == os.lstat(v1 / "same.bin").st_ino
    for n in ("flip.bin", "grow.bin", "cut.bin", "mode.bin"):
        assert os.lstat(v2 / n).st_ino != os.lstat(v1 / n).st_ino, n
    assert not (v2 / "gone.bin").exists()
    assert st["files_linked"] == 1 and st["bytes_linked"] == sizes["same.bin"], st
    # flip: all but block 1; grow and cut: block 0; mode: every block (same bytes, the metadata differs)
    assert st["files_backfilled"] == 4, st
    assert st["bytes_backfilled"] == (sizes["flip.bin"] - BB) + BB + BB + sizes["mode.bin"], st
    assert st["bytes_written"] == BB + (100 + MiB) + 5 + (BB + 3), st
    assert st["files_base_untrusted"] == 0 and st["lanes_used"] >= lanes, st
    _check(vm, orc, src, v2, t2)
    assert _state(v1) == before
    _restores(vm, orc, v1, t1, ref1)


# ------------------------------------------------------------------------------------------ hard-link structure
def test_base_hard_link_pair_does_not_join_separate_source_files(vm, orc, shm_tmp):
    src1, src2, v1, v2 = shm_tmp / "src1", shm_tmp / "src2", shm_tmp / "v1", shm_tmp / "v2"
    src1.mkdir(), src2.mkdir()
    body = orc.splitmix_bytes(9, BB + 3).tobytes()
    t = 1_600_000_000_000_000_000
    (src1 / "a").write_bytes(body)
    os.link(src1 / "a", src1 / "b")
    (src1 / "c").write_bytes(b"c" * 100)
    for n in ("a", "b"):                       # the same bytes, now two files
        (src2 / n).write_bytes(body)
    (src2 / "c").write_bytes(b"c" * 100)
    for p in (src1 / "a", src1 / "c", src2 / "a", src2 / "b", src2 / "c"):
        os.utime(p, ns=(t, t))
    _snap(vm, src1, v1)
    st, t2 = _snap(vm, src2, v2, v1)
    assert os.lstat(v2 / "a").st_ino != os.lstat(v2 / "b").st_ino
    assert os.lstat(v1 / "a").st_ino == os.lstat(v1 / "b").st_ino
    assert st["files_linked"] == 2, st        # a (to the pair's inode, once) and c
    _check(vm, orc, src2, v2, t2)


# ------------------------------------------------------------------------------------------ untrusted base
def _three(orc, src: Path):
    src.mkdir()
    for i in range(3):
        (src / f"f{i}.bin").write_bytes(orc.splitmix_bytes(60 + i, BB + 1000 * i).tobytes())


def test_base_file_rewritten_out_of_band_is_copied_from_the_source(vm, orc, shm_tmp):
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    _three(orc, src)
    _snap(vm, src, v1)
    time.sleep(0.05)
    p = v1 / "f1.bin"
    old = os.lstat(p)
    p.write_bytes(orc.splitmix_bytes(99, old.st_size).tobytes())       # same inode, same size, other bytes ...
    os.utime(p, ns=(old.st_atime_ns, old.st_mtime_ns))                  # ... and the mtime put back
    st, t2 = _snap(vm, src, v2, v1)
    assert st["files_base_untrusted"] == 1 and st["files_linked"] == 2, st
    assert os.lstat(v2 / "f1.bin").st_ino != p.stat().st_ino
    _check(vm, orc, src, v2, t2)


def test_base_table_written_for_another_directory(vm, orc, shm_tmp):
    """A version directory whose blocks.vmig was last written by a hand-off copy into the container's layer, not for
    diff/: no file of the base is trusted, the snapshot is a plain copy."""
    src, v1, v2, layer = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2", shm_tmp / "layer"
    _three(orc, src)
    _snap(vm, src, v1)
    layer.mkdir()
    vm.migrate_tree(src, layer, None, shm_tmp / "v1.vmig")
    st, t2 = _snap(vm, src, v2, v1)
    assert st["files_linked"] == 0 and st["files_backfilled"] == 0 and st["files_base_untrusted"] == 3, st
    assert st["bytes_written"] == st["bytes_total"]
    _check(vm, orc, src, v2, t2)


def test_base_on_another_filesystem(vm, orc, shm_tmp, tmp_path):
    if os.stat(shm_tmp).st_dev == os.stat(tmp_path).st_dev:
        pytest.skip("needs /dev/shm and the test's temporary directory on two filesystems")
    src, v1, v2 = shm_tmp / "src", tmp_path / "v1", shm_tmp / "v2"
    _three(orc, src)
    _snap(vm, src, v1)
    st, t2 = _snap(vm, src, v2, v1)
    assert st["files_linked"] == 0 and st["files_backfilled"] == 0 and st["bytes_written"] == st["bytes_total"], st
    _check(vm, orc, src, v2, t2)


# ------------------------------------------------------------------------------------------ chain
def test_chain_survives_the_removal_of_its_first_snapshot(vm, orc, shm_tmp):
    src = shm_tmp / "src"
    _three(orc, src)
    (src / "big.bin").write_bytes(orc.splitmix_bytes(70, 3 * BB + 11).tobytes())
    v = [shm_tmp / f"v{i}" for i in (1, 2, 3)]
    refs, tables = [], []
    for i, snap in enumerate(v):
        if i == 1:
            _flip(src / "big.bin", 2 * BB + 3)
            (src / "f2.bin").unlink()
        if i == 2:
            _flip(src / "big.bin", 10)
            (src / "added.bin").write_bytes(b"a" * 7000)
        st, t = _snap(vm, src, snap, v[i - 1] if i else None)
        if i:
            assert st["files_linked"] >= 1 and st["files_backfilled"] >= 1, st
        refs.append(_check(vm, orc, src, snap, t))
        tables.append(t)
    shutil.rmtree(v[0])
    for snap, t, ref in zip(v[1:], tables[1:], refs[1:]):
        _restores(vm, orc, snap, t, ref)
        st = vm.restore_tree(snap, t, None, flags=vm.F_HASH_ONLY)
        assert st["bytes_written"] == 0


# ------------------------------------------------------------------------------------------ O_DIRECT
def test_direct_io_backfill_of_a_partial_last_sector(vm, orc, tmp_path):
    src, v1, v2 = tmp_path / "src", tmp_path / "v1", tmp_path / "v2"
    src.mkdir()
    size = 2 * BB + 1000                                   # the backfilled last block ends inside a sector
    (src / "d.bin").write_bytes(orc.splitmix_bytes(80, size).tobytes())
    (src / "e.bin").write_bytes(orc.splitmix_bytes(81, BB + 512).tobytes())
    _snap(vm, src, v1, flags=vm.F_VERIFY | vm.F_DIRECT_IO)
    _flip(src / "d.bin", 5)
    os.chmod(src / "e.bin", 0o640)
    st, t2 = _snap(vm, src, v2, v1, flags=vm.F_VERIFY | vm.F_DIRECT_IO)
    assert st["files_backfilled"] == 2 and st["bytes_backfilled"] == (size - BB) + BB + 512, st
    assert (v2 / "d.bin").read_bytes() == (src / "d.bin").read_bytes()
    assert (v2 / "e.bin").stat().st_size == BB + 512
    _check(vm, orc, src, v2, t2)


# ------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_destination_untouched(vm, orc, shm_tmp):
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    _three(orc, src)
    _, t1 = _snap(vm, src, v1)
    v2.mkdir()
    (v1 / "inner").mkdir()
    out = shm_tmp / "v2.vmig"
    before = _state(v1)

    def refused(code, **kw):
        args = dict(base=v1, base_table=t1, out_table=out)
        args.update(kw.pop("args", {}))
        with pytest.raises(vm.VmigError) as ei:
            vm.snapshot_tree(src, kw.pop("dst", v2), args["base"], args["base_table"], args["out_table"], **kw)
        assert ei.value.code == code, ei.value

    refused(vm.VMIG_ETABLE, block_bytes=MiB)
    refused(vm.VMIG_EINVAL, args=dict(base_table=None))
    refused(vm.VMIG_EINVAL, args=dict(base=None))
    refused(vm.VMIG_EINVAL, args=dict(out_table=None))
    for f in (vm.F_MOVE_SRC, vm.F_HASH_ONLY, vm.F_CUFILE):
        refused(vm.VMIG_EINVAL, flags=f)
    refused(vm.VMIG_EINVAL, dst=v1)
    refused(vm.VMIG_EINVAL, dst=v1 / "inner")
    assert os.listdir(v2) == [] and not out.exists() and _state(v1) == before


# ------------------------------------------------------------------------------------------ hand-off
def test_handoff_incremental_snapshots_and_rollbacks(vm, orc, shm_tmp):
    import importlib
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {f"rs-{i}": shm_tmp / f"upper_{i}" for i in (2, 3, 4, 5)}
    for p in ups.values():
        p.mkdir()
    for i in range(3):
        (ups["rs-2"] / f"g{i}.bin").write_bytes(orc.splitmix_bytes(300 + i, 9 * MiB + i).tobytes())
    ref2 = shm_tmp / "ref2"
    ref2.mkdir()
    orc.ref_copy(ups["rs-2"], ref2)
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        (ho.versionDir("rs-1") / "diff").mkdir(parents=True)        # a version without its table is never a base
        assert ho.baseVersion("rs-2") is None
        st2 = ho.SnapshotVersionIncremental("rs-2")
        assert st2.get("files_linked", 0) == 0 and st2["bytes_written"] == st2["bytes_total"]
        orc.ref_copy(ups["rs-2"], ups["rs-3"])
        _flip(ups["rs-3"] / "g1.bin", 5 * MiB)
        ref3 = shm_tmp / "ref3"
        ref3.mkdir()
        orc.ref_copy(ups["rs-3"], ref3)
        assert ho.baseVersion("rs-3") == "rs-2"
        st3 = ho.SnapshotVersionIncremental("rs-3")
        assert st3["files_linked"] == 2 and st3["files_backfilled"] == 1 and st3["bytes_written"] == BB, st3
        ho.RollbackFromSnapshot("rs-2", "rs-4")
        ho.RollbackFromSnapshot("rs-3", "rs-5")
        assert orc.compare_trees(ref2, ups["rs-4"]) == [] and orc.compare_trees(ref3, ups["rs-5"]) == []
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)


# ------------------------------------------------------------------------------------------ bench scale
def _free_bytes(p) -> int:
    st = os.statvfs(p)
    avail = [st.f_bavail * st.f_frsize]
    for line in Path("/proc/meminfo").read_text().splitlines():
        if line.startswith("MemAvailable:"):
            avail.append(int(line.split()[1]) * 1024)
    return min(avail)


def test_unchanged_10x1GiB_layer_takes_no_new_space(vm, orc, shm_tmp):
    n_files, fbytes = 10, 1 << 30
    if _free_bytes(shm_tmp) < 2.5 * n_files * fbytes:
        pytest.skip("needs ~25 GiB of tmpfs for a 10 x 1 GiB layer and its snapshot")
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    src.mkdir()
    vm.datagen_files(src, 0x5EED, n_files, fbytes)
    _snap(vm, src, v1)
    s0 = os.statvfs(shm_tmp)
    st, t2 = _snap(vm, src, v2, v1)
    s1 = os.statvfs(shm_tmp)
    grew = (s0.f_bfree - s1.f_bfree) * s0.f_frsize
    assert st["bytes_written"] == 0 and st["files_linked"] == n_files and st["blocks_skipped"] == 2560, st
    assert grew < 8 * MiB, grew
    assert (vm.table_hashes(t2) == vm.table_hashes(v1.with_name("v1.vmig"))).all()
