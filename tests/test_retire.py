"""vmig_retire_versions on the GPU (-m gpu): old versions of a snapshot store (built as tests/test_scrub.py builds one)
are removed while the kept versions' tables stay trusted, so the next incremental snapshot links what it linked before.

rm -rf of a version moves the ctime of every inode it shared with the kept versions; the tests show that gap first, then
that the retire closes it without trusting anything it did not re-read: every re-recorded identity is the file's own,
every kept table differs only in identity fields, and the kept versions still scrub clean and restore as the tar pipe
copies them."""
import importlib
import os
import shutil
import struct
import time
from pathlib import Path

import pytest

from test_scrub import BB, Canceller, _disk_dir, _fds, _flip, _source, _threads, build_store, read_table, regular_files

pytestmark = pytest.mark.gpu
MiB = 1 << 20


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def identity_bytes(raw: bytes) -> set:
    """Offsets of the ino / ctime_ns bytes of every record of a VMIGBT02 table (include/vmig.h)."""
    assert raw[:8] == b"VMIGBT02"
    (nf,) = struct.unpack_from("<Q", raw, 16)
    off, out = 32, set()
    for _ in range(nf):
        (pl,) = struct.unpack_from("<I", raw, off)
        off += 4 + pl
        out.update(range(off + 16, off + 32))
        off += 32
    return out


def differs_only_in_identities(old: bytes, new: bytes) -> bool:
    ids = identity_bytes(old)
    return len(old) == len(new) and all(i in ids for i in range(len(old)) if old[i] != new[i])


def unchanged_source_files(src: Path) -> int:
    return sum(1 for st in regular_files(src).values() if st.st_nlink == 1 and st.st_size > 0)


def identities_match_the_files(d: Path, t: Path) -> bool:
    for rel, (_size, _h, ino, ct) in read_table(t).items():
        if ino:
            st = os.lstat(d / rel)
            if (st.st_ino, st.st_ctime_ns) != (ino, ct):
                return False
    return True


def unlink_moves_ctime(d: Path) -> bool:
    """Whether removing one hard link of an inode moves the inode's ctime on d's filesystem (Linux tmpfs, ext4 and xfs
    do; some sandboxed filesystems do not)."""
    probe = d / "ctime_probe"
    probe.mkdir()
    (probe / "a").write_bytes(b"x")
    os.link(probe / "a", probe / "b")
    before = os.stat(probe / "a").st_ctime_ns
    time.sleep(0.01)
    (probe / "b").unlink()
    moved = os.stat(probe / "a").st_ctime_ns != before
    shutil.rmtree(probe)
    return moved


def move_ctimes(dirs):
    """Move the ctime of every regular file under dirs and nothing else (utime to its own times): what unlinking those
    paths does to the inodes they share with the kept versions, where the filesystem's unlink moves ctimes."""
    for d in dirs:
        for dp, _dns, fns in os.walk(d):
            for n in fns:
                p = os.path.join(dp, n)
                st = os.lstat(p)
                if os.path.isfile(p) and not os.path.islink(p):
                    os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns))


def as_unlink_would(shm_tmp: Path, dirs):
    """The tests need the kept records the removal leaves stale on Linux filesystems; where unlink leaves ctimes alone,
    the retired versions' files get their ctime moved by hand before the removal, so the data path is the same."""
    if not unlink_moves_ctime(shm_tmp):
        move_ctimes(dirs)


def next_snapshot(vm, root: Path, base):
    v = root / "next"
    v.mkdir()
    return vm.snapshot_tree(root / "src", v, base[0], base[1], root / "next.vmig")


# ------------------------------------------------------------------------------------------ 1. the gap, closed
def test_retire_keeps_the_next_snapshot_incremental(vm, orc, shm_tmp):
    A, B = build_store(vm, orc, shm_tmp / "A"), build_store(vm, orc, shm_tmp / "B")
    tar = {}
    for k in (2, 3):
        tar[k] = shm_tmp / f"tar{k}"
        tar[k].mkdir()
        orc.ref_copy(B[k][0], tar[k])

    as_unlink_would(shm_tmp, [d for d, _ in A[:2] + B[:2]])
    # rm -rf: the next snapshot no longer trusts what the removed versions shared, and copies it
    for d, t in A[:2]:
        shutil.rmtree(d)
        t.unlink()
    st = next_snapshot(vm, shm_tmp / "A", A[3])
    assert st["files_base_untrusted"] > 0 and st["bytes_written"] > 0, st

    before = {t: t.read_bytes() for _, t in B[2:]}
    r = vm.retire_versions(B[:2], B[2:])
    assert r["versions_retired"] == 2 and r["tables_rewritten"] == 2, r
    assert r["records_stale"] > 0 and r["records_restamped"] == r["records_stale"], r
    assert r["stats"]["bytes_h2d"] == r["bytes_rehashed"] > 0
    assert not any(p.exists() for pair in B[:2] for p in pair)
    for d, t in B[2:]:
        assert identities_match_the_files(d, t), t
        assert differs_only_in_identities(before[t], t.read_bytes()) and before[t] != t.read_bytes(), t
    assert vm.scrub_store(B[2:])["verdicts"] == [vm.VMIG_OK] * 2
    for k in (2, 3):
        dst = shm_tmp / f"restored{k}"
        dst.mkdir()
        vm.restore_tree(B[k][0], B[k][1], dst)
        assert orc.compare_trees(tar[k], dst) == [], k

    st = next_snapshot(vm, shm_tmp / "B", B[3])
    assert st["files_linked"] == unchanged_source_files(shm_tmp / "B" / "src"), st
    assert st["bytes_written"] == 0 and st["files_base_untrusted"] == 0, st


# ------------------------------------------------------------------------------------------ 2. freed bytes
def test_freed_bytes_are_the_inodes_whose_every_link_is_retired(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp / "s")
    held = shm_tmp / "held.bin"
    os.link(pairs[0][0] / "big.bin", held)                 # v1's own big.bin, also linked outside the store
    links = {}
    for d, _ in pairs[:2]:
        for dp, _dns, fns in os.walk(d):
            for n in fns:
                s = os.lstat(os.path.join(dp, n))
                if os.path.isfile(os.path.join(dp, n)) and not os.path.islink(os.path.join(dp, n)):
                    k = links.setdefault((s.st_dev, s.st_ino), [s.st_nlink, 0, s.st_size])
                    k[1] += 1
    freed = [size for nlink, seen, size in links.values() if nlink == seen]
    entries = sum(len(dns) + len(fns) for d, _ in pairs[:2] for _dp, dns, fns in os.walk(d))
    r = vm.retire_versions(pairs[:2], pairs[2:])
    assert (r["files_freed"], r["bytes_freed"]) == (len(freed), sum(freed)), r
    assert r["entries_removed"] == entries and r["versions_retired"] == 2, r
    assert not any(p.exists() for pair in pairs[:2] for p in pair)
    assert held.read_bytes()[:4096] == (pairs[2][0] / "big.bin").read_bytes()[:4096] and os.stat(held).st_nlink == 1


# ------------------------------------------------------------------------------------------ 3. no laundering
def test_a_changed_inode_is_not_restamped(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp / "s")
    (v3, t3), (v4, t4) = pairs[2:]
    assert os.stat(v3 / "exact.bin").st_nlink == 4
    _flip(pairs[0][0] / "exact.bin", 12345, keep_mtime=True)          # rewritten in place, shared by v3 and v4
    body = (v4 / "data" / "keep.bin").read_bytes()
    (v4 / "data" / "keep.tmp").write_bytes(body)
    os.replace(v4 / "data" / "keep.tmp", v4 / "data" / "keep.bin")    # v4's keep.bin: a new inode, the same bytes
    old3, old4 = read_table(t3), read_table(t4)
    as_unlink_would(shm_tmp, [d for d, _ in pairs[:2]])
    r = vm.retire_versions(pairs[:2], pairs[2:])
    assert r["records_stale"] - r["records_restamped"] == 2, r
    new3, new4 = read_table(t3), read_table(t4)
    assert new3["exact.bin"] == old3["exact.bin"] and new4["exact.bin"] == old4["exact.bin"]
    assert new4["data/keep.bin"] == old4["data/keep.bin"]              # another inode: not stale, untouched
    assert new3["data/keep.bin"][2:] == (os.stat(v3 / "data" / "keep.bin").st_ino, os.stat(v3 / "data" / "keep.bin").st_ctime_ns)
    for t, new in ((t3, new3), (t4, new4)):
        for rel, rec in new.items():
            if rel != "exact.bin" and not (t == t4 and rel == "data/keep.bin") and rec[2]:
                st = os.lstat((v3 if t == t3 else v4) / rel)
                assert rec[2:] == (st.st_ino, st.st_ctime_ns), (t, rel)
    s = vm.scrub_store(pairs[2:])
    assert {(f["version"], f["kind"], f["path"], f["block"]) for f in s["findings"]} == {(0, "block", "exact.bin", 0), (1, "block", "exact.bin", 0)}


# ------------------------------------------------------------------------------------------ 4. cancel and re-run
def _datagen_store(vm, root: Path):
    src = root / "src"
    src.mkdir(parents=True)
    vm.datagen_files(src, 77, 6, 256 * MiB)
    pairs = []
    for k in (1, 2, 3):
        if k > 1:
            _flip(src / f"f0000{k}.bin", 3)
        d, t = root / f"v{k}", root / f"v{k}.vmig"
        d.mkdir()
        vm.snapshot_tree(src, d, *(pairs[-1] if pairs else (None, None)), t)
        pairs.append((d, t))
    return pairs


def test_cancel_in_the_data_pass_then_rerun(vm, orc, shm_tmp):
    pairs = _datagen_store(vm, shm_tmp)
    vm.scrub_store(pairs[1:])                                # warms the pipes: the thread / fd baseline
    threads, fds = _threads(), _fds()
    kept = {t: t.read_bytes() for _, t in pairs[1:]}
    as_unlink_would(shm_tmp, [pairs[0][0]])
    with vm.Ctl() as c:
        k = Canceller(c, lambda p: p["phase_name"] == "DATA" and p["bytes_total"] and p["bytes_hashed"] >= 0.5 * p["bytes_total"])
        k.start()
        try:
            vm.retire_versions(pairs[:1], pairs[1:], ctl=c)
            res = None
        except vm.VmigError as e:
            res = e
        k.done.set()
        k.join()
        assert k.fired and res is not None and res.code == vm.VMIG_ECANCELED, res
        assert c.progress()["phase_name"] == "DATA"
    assert not pairs[0][0].exists() and not pairs[0][1].exists()
    assert {t: t.read_bytes() for _, t in pairs[1:]} == kept
    assert not [n for n in os.listdir(shm_tmp) if ".tmp" in n]
    r = vm.retire_versions([], pairs[1:])
    assert r["versions_retired"] == 0 and r["records_restamped"] == r["records_stale"] > 0 and r["tables_rewritten"] == 2, r
    st = next_snapshot(vm, shm_tmp, pairs[2])
    assert st["files_linked"] == 6 and st["bytes_written"] == 0 and st["files_base_untrusted"] == 0, st
    assert _threads() == threads and _fds() == fds


def test_cancel_in_the_removal_then_rerun(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp / "s", n_versions=3)
    many = pairs[0][0] / "many"
    for i in range(200):
        (many / f"d{i:03d}").mkdir(parents=True)
        for j in range(250):
            (many / f"d{i:03d}" / f"f{j:03d}").touch()
    vm.scrub_store(pairs[1:])
    threads, fds = _threads(), _fds()
    with vm.Ctl() as c:
        k = Canceller(c, lambda p: p["phase_name"] == "UNLINK")
        k.start()
        try:
            vm.retire_versions(pairs[:1], pairs[1:], ctl=c)
            res = None
        except vm.VmigError as e:
            res = e
        k.done.set()
        k.join()
        assert k.fired and res is not None and res.code == vm.VMIG_ECANCELED, res
        assert c.progress()["phase_name"] == "UNLINK"
    assert pairs[0][0].is_dir() and not pairs[0][1].exists()         # half removed, its table already gone
    r = vm.retire_versions(pairs[:1], pairs[1:])
    assert r["versions_retired"] == 1 and not pairs[0][0].exists(), r
    assert all(identities_match_the_files(d, t) for d, t in pairs[1:])
    assert _threads() == threads and _fds() == fds


# ------------------------------------------------------------------------------------------ 5. safety
def test_retire_never_leaves_the_retired_trees(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp / "s", n_versions=3)
    outside = shm_tmp / "outside"
    (outside / "inner").mkdir(parents=True)
    (outside / "inner" / "f").write_bytes(b"keep me")
    os.symlink(outside, pairs[0][0] / "sub" / "to_outside")
    os.symlink(pairs[2][0], shm_tmp / "s" / "alias")
    kept_raw = {t: t.read_bytes() for _, t in pairs[1:]}
    other = shm_tmp / "other_bb.vmig"
    vm.manifest(pairs[2][0], other, block_bytes=1 << 20)
    cases = [(vm.VMIG_ENOTDIR, [(shm_tmp / "s" / "alias", shm_tmp / "alias.vmig")], pairs[1:]),
             (vm.VMIG_EINVAL, [pairs[0]], [pairs[0], pairs[1]]),
             (vm.VMIG_EINVAL, [(pairs[1][0] / "sub", shm_tmp / "x.vmig")], pairs[1:]),
             (vm.VMIG_ETABLE, pairs[:1], [pairs[1], (pairs[2][0], other)])]
    for code, retire, keep in cases:
        with pytest.raises(vm.VmigError) as ei:
            vm.retire_versions(retire, keep)
        assert ei.value.code == code, (code, ei.value)
        assert pairs[0][1].exists() and (pairs[0][0] / "sub" / "to_outside").is_symlink() and pairs[2][0].is_dir()
    assert {t: t.read_bytes() for _, t in pairs[1:]} == kept_raw
    vm.retire_versions(pairs[:1], pairs[1:])
    assert not pairs[0][0].exists() and (outside / "inner" / "f").read_bytes() == b"keep me"


# ------------------------------------------------------------------------------------------ 6. lanes and O_DIRECT
@pytest.mark.parametrize("mode", ["3lanes", "direct"])
def test_same_tables_with_three_lanes_and_direct_io(vm, orc, shm_tmp, tmp_path, mode):
    root = _disk_dir(tmp_path) if mode == "direct" else shm_tmp
    pairs = build_store(vm, orc, root / "s")
    move_ctimes([pairs[0][0]])                     # every version's records of what v1 shares go stale
    raw = {t: t.read_bytes() for _, t in pairs}
    plain = vm.retire_versions([], pairs)
    assert plain["records_restamped"] > 0, plain
    want = {t: t.read_bytes() for _, t in pairs}
    for t, b in raw.items():
        t.write_bytes(b)
    kw = {"lanes_per_gpu": 3} if mode == "3lanes" else {"flags": vm.F_DIRECT_IO}
    other = vm.retire_versions([], pairs, **kw)
    assert {t: t.read_bytes() for _, t in pairs} == want
    assert other["records_restamped"] == plain["records_restamped"]
    if mode == "3lanes":
        assert other["stats"]["lanes_used"] == 3
    else:
        assert other["stats"]["files_direct"] > 0


# ------------------------------------------------------------------------------------------ 7. hand-off
def _sequence(vm, orc, ho, root: Path, ups: dict, retire: bool):
    ho.set_merges_root(root)
    written = []
    for v in range(2, 10):
        name = f"rs-{v}"
        written.append(ho.SnapshotVersionIncremental(name)["bytes_written"])
        if retire and v == 3:
            (ho.versionDir("rs-1") / "diff").mkdir(parents=True)       # a snapshot that failed before its table
        if retire:
            out = ho.RetireVersions("rs", keep=2)
            assert out["kept"] == [f"rs-{k}" for k in range(max(2, v - 1), v + 1)], out
    return written


def test_retire_replicaset_keeps_the_newest_two(vm, orc, shm_tmp):
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {f"rs-{v}": shm_tmp / "up" / f"rs-{v}" for v in range(2, 10)}
    _source(orc, ups["rs-2"])
    for v in range(3, 10):
        ups[f"rs-{v}"].mkdir(parents=True)
        orc.ref_copy(ups[f"rs-{v - 1}"], ups[f"rs-{v}"])
        _flip(ups[f"rs-{v}"] / "data" / "g2.bin", v * BB + 5)
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    try:
        (shm_tmp / "A" / "merges" / "rs" / "rs-0").mkdir(parents=True)      # the running container's table only
        (shm_tmp / "A" / "merges" / "rs" / "rs-0" / "blocks.vmig").write_bytes(b"not a snapshot")
        with_retire = _sequence(vm, orc, ho, shm_tmp / "A", ups, True)
        without = _sequence(vm, orc, ho, shm_tmp / "B", ups, False)
        assert with_retire == without
        assert sorted(os.listdir(shm_tmp / "A" / "merges" / "rs")) == ["rs-0", "rs-8", "rs-9"]
        assert (shm_tmp / "A" / "merges" / "rs" / "rs-0" / "blocks.vmig").read_bytes() == b"not a snapshot"
        ho.set_merges_root(shm_tmp / "A")
        for name in ("rs-8", "rs-9"):
            d, t = ho.snapshotPaths(name)
            dst, tar = shm_tmp / f"restored-{name}", shm_tmp / f"tar-{name}"
            dst.mkdir()
            tar.mkdir()
            vm.restore_tree(d, t, dst)
            orc.ref_copy(ups[name], tar)
            assert orc.compare_trees(tar, dst) == [], name
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
