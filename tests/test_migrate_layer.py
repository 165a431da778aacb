"""vmig_migrate_layer on the GPU (-m gpu).  Every paused pass is held to vmig_migrate_tree on a destination filled from the
same source by its own live pass: the same tree, the same out table (paths, sizes, hashes), the same bytes written, and
both to the tar copy of the source.  The bytes read from the source are restated here from the two tables and lstat."""
import importlib
import os
import stat
import threading
import time
from pathlib import Path

import pytest

import _layer_model as lm
from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _flip(p: Path, off: int):
    with open(p, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x5A]))


def _settle():
    """Past the coarse clock's tick: a file written just before a live pass is recorded only once its ctime is older
    than the clock reading taken before its first read (include/vmig.h, src_out_table)."""
    time.sleep(0.05)


def _populate(root: Path, orc, bb: int):
    for d in ("m", "u"):
        (root / d).mkdir()
    sizes = {"m/a.bin": 5 * bb + 123, "m/b.bin": 3 * bb, "m/c.bin": 4 * bb + 7, "m/d.bin": 2 * bb + 11, "m/e.bin": 3 * bb + 1,
             "u/chmod.bin": 2 * bb, "u/todir.bin": bb + 3}
    sizes.update({f"u/keep{i}.bin": (i + 1) * bb + 17 * i for i in range(4)})
    for i, (rel, n) in enumerate(sorted(sizes.items())):
        (root / rel).write_bytes(lm.data(40 + i, n))
    (root / "u" / "hl_old").write_bytes(lm.data(60, bb + 9))          # a hard-link pair the live pass already sees
    os.link(root / "u" / "hl_old", root / "u" / "hl_old2")
    (root / "rich").mkdir()
    make_rich_tree(root / "rich", orc, big=2 * bb + 777)


def _edit(root: Path, bb: int):
    """What the tenant does between the live pass and the paused one."""
    _flip(root / "m" / "a.bin", 2 * bb + 5)                                    # in-place write
    with open(root / "m" / "b.bin", "ab") as f:                                # append
        f.write(lm.data(90, bb // 2 + 3))
    os.truncate(root / "m" / "c.bin", 2 * bb + 5)                              # truncate
    os.unlink(root / "m" / "d.bin")                                            # deletion
    (root / "n").mkdir()
    os.rename(root / "m" / "e.bin", root / "n" / "e_moved.bin")                # rename
    (root / "n" / "new1.bin").write_bytes(lm.data(91, 2 * bb + 9))             # new file
    os.chmod(root / "u" / "chmod.bin", 0o600)                                  # chmod only: read, nothing written
    (root / "n" / "hl_a").write_bytes(lm.data(94, bb + 2))                     # new hard-link pair
    os.link(root / "n" / "hl_a", root / "n" / "hl_b")
    os.symlink("../m/a.bin", root / "n" / "sym")
    os.mkfifo(root / "n" / "fifo")
    (root / "n" / "empty").write_bytes(b"")
    os.unlink(root / "u" / "todir.bin")                                        # a file replaced by a directory
    (root / "u" / "todir.bin").mkdir()
    (root / "u" / "todir.bin" / "inner").write_bytes(lm.data(95, 77))


UNTOUCHED = [b"u/keep0.bin", b"u/keep1.bin", b"u/keep2.bin", b"u/keep3.bin"]


def _regular_primaries(root: Path):
    """rel (bytes) -> lstat of each regular file that is the first path (bytewise) of its in-tree inode group."""
    root = os.fsencode(os.fspath(root))
    seen, out, paths = set(), {}, []
    for dp, _, fns in os.walk(root):
        for n in fns:
            paths.append(os.path.relpath(os.path.join(dp, n), root))
    for rel in sorted(paths):
        st = os.lstat(os.path.join(root, rel))
        if stat.S_ISREG(st.st_mode) and st.st_ino not in seen:
            seen.add(st.st_ino)
            out[rel] = st
    return out


def _records(vm, orc, table):
    t, h = orc.read_table(table), vm.table_hashes(table)
    return {rel: (size, first, ino, ct) for (rel, size, first), (ino, ct) in zip(t["entries"], t["identity"])}, h


def _dst_trusted(dst: Path, rel: bytes, p) -> bool:
    """The prior table still vouches for the destination file (the in-place diff path's rule)."""
    try:
        ds = os.lstat(os.path.join(os.fsencode(os.fspath(dst)), rel))
    except (FileNotFoundError, NotADirectoryError):         # nothing there, or a file where the source has a directory
        return False
    return bool(p and p[2] and stat.S_ISREG(ds.st_mode) and ds.st_nlink == 1 and
                (ds.st_ino, ds.st_size, ds.st_ctime_ns) == (p[2], p[0], p[3]))


def expected_verified(vm, orc, src: Path, dst: Path, prior, bb: int) -> int:
    """Bytes F_VERIFY re-reads, by include/vmig.h: every destination file the call creates or replaces, writes a block
    into, or resizes -- all but those patched in place whose size and every block hash stay the prior record's.  Taken
    before the call."""
    prec, ph = _records(vm, orc, prior)
    entries, hashes = orc.block_table_of_tree(src, bb)
    first = {rel: f for rel, _, f in entries}
    n = 0
    for rel, st in _regular_primaries(src).items():
        p = prec.get(rel)
        nb = -(-st.st_size // bb)
        kept = (_dst_trusted(dst, rel, p) and p[0] == st.st_size and
                all(int(ph[p[1] + i]) == int(hashes[first[rel] + i]) for i in range(nb)))
        n += 0 if kept else st.st_size
    return n


def expected_read(vm, orc, src: Path, src_table, dst: Path, prior, bb: int) -> dict:
    """rel -> source bytes the call reads, by include/vmig.h: a trusted source file reads the blocks of its record that
    are not the prior record's (hash, length) at the same index of a destination file the prior table still vouches
    for; every other regular file is read in full.  Taken before the call."""
    srec, sh = _records(vm, orc, src_table)
    prec, ph = _records(vm, orc, prior) if prior else ({}, None)
    out = {}
    for rel, st in _regular_primaries(src).items():
        if not st.st_size:
            continue
        r = srec.get(rel)
        if not (r and r[2] and (st.st_ino, st.st_size, st.st_ctime_ns) == (r[2], r[0], r[3])):
            out[rel] = st.st_size
            continue
        p = prec.get(rel)
        dtrust = _dst_trusted(dst, rel, p)
        n = 0
        for i in range(-(-st.st_size // bb)):
            ln = min(bb, st.st_size - i * bb)
            if dtrust and i * bb < p[0] and min(bb, p[0] - i * bb) == ln and int(ph[p[1] + i]) == int(sh[r[1] + i]):
                continue
            n += ln
        out[rel] = n
    return out


def src_state(root: Path) -> dict:
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in [""] + dns + fns:
            p = os.path.join(dp, n) if n else dp
            st = os.lstat(p)
            body = Path(p).read_bytes() if stat.S_ISREG(st.st_mode) else st.st_size
            out[p] = (st.st_ino, st.st_mode, st.st_mtime_ns, st.st_ctime_ns, body)
    return out


def same_tree(orc, a, b):
    assert lm.diff_manifests(lm.tree_in_itself(orc, a), lm.tree_in_itself(orc, b)) == []


def _no_tmp(*tables):
    for t in tables:
        assert not [n for n in os.listdir(t.parent) if n.startswith(t.name + ".tmp")], t


# ------------------------------------------------------------------------------------------ 1. equivalence
def _paused_pass(vm, orc, root: Path, s: Path, src_table, dA, dB, tA, tB, tag: str, flags: int, bb: int, lanes: int) -> dict:
    """migrate_layer(s, src_table, dA, prior tA) next to migrate_tree(s, dB, prior tB): the same tree, table and bytes
    written, both the tar copy of s; the bytes read and re-read as include/vmig.h states them.  Returns rel -> bytes read."""
    want = expected_read(vm, orc, s, src_table, dA, tA, bb)
    want_verified = expected_verified(vm, orc, s, dA, tA, bb)
    before = src_state(s)
    tables = {p: p.read_bytes() for p in (tA, src_table)}
    tA2, tB2 = root / f"tA{tag}.vmig", root / f"tB{tag}.vmig"
    rB = vm.migrate_tree(s, dB, tB, tB2, flags=flags, block_bytes=bb, lanes_per_gpu=lanes)
    rA = vm.migrate_layer(s, src_table, dA, tA, tA2, None, flags=flags, block_bytes=bb, lanes_per_gpu=lanes)
    assert src_state(s) == before and all(p.read_bytes() == b for p, b in tables.items())
    assert rA["bytes_read"] == sum(want.values()) and rA["files_read"] == sum(1 for v in want.values() if v), (rA, want)
    assert rA["files_trusted"] > 0 and rA["files_unread"] > 0 and rA["src_recorded"] == rA["src_unrecorded"] == 0
    assert rA["bytes_total"] == rA["bytes_read"] and rA["bytes_written"] == rB["bytes_written"], (rA, rB)
    assert rA["pruned"] == rB["pruned"] and rA["files_untrusted"] == rB["files_untrusted"]
    if flags & vm.F_VERIFY:
        assert rA["bytes_h2d"] == rA["bytes_read"] + rA["bytes_verified"]
        assert 0 < rA["bytes_verified"] == want_verified < rB["bytes_total"], (rA, want_verified)
    else:
        assert rA["bytes_h2d"] == rA["bytes_read"] and rA["files_verified"] == 0
    same_tree(orc, dA, dB)
    tar = root / f"tar{tag}"
    tar.mkdir()
    orc.ref_copy(s, tar)
    assert orc.compare_trees(tar, dA) == [] and orc.compare_trees(tar, dB) == []
    a2, b2 = orc.read_table(tA2), orc.read_table(tB2)
    assert a2["entries"] == b2["entries"] and (vm.table_hashes(tA2) == vm.table_hashes(tB2)).all()
    _, want_hashes = orc.block_table_of_tree(s, bb)
    assert (vm.table_hashes(tA2) == want_hashes).all()
    _no_tmp(tA2, tB2)
    return want


@pytest.mark.parametrize("bb,lanes,disk", [(4 << 20, 1, False), (65536, 3, False), (4 << 20, 3, True)])
def test_layer_migration_equals_tree_migration(vm, orc, shm_tmp, tmp_path, bb, lanes, disk):
    root = tmp_path if disk else shm_tmp
    direct = vm.F_DIRECT_IO if disk else 0
    src0 = root / "src0"
    src0.mkdir()
    _populate(src0, orc, bb)
    for verify in (vm.F_VERIFY, 0):
        k = "v" if verify else "n"
        s, dA, dB = root / f"src{k}", root / f"dA{k}", root / f"dB{k}"
        lm.freeze(src0, s)
        dA.mkdir(), dB.mkdir()
        tA1, sA1, tB1 = root / f"tA1{k}.vmig", root / f"sA1{k}.vmig", root / f"tB1{k}.vmig"
        _settle()
        # pass 1 (live) on each side
        r1 = vm.migrate_layer(s, None, dA, None, tA1, sA1, flags=vm.F_VERIFY | direct, block_bytes=bb, lanes_per_gpu=lanes)
        vm.migrate_tree(s, dB, None, tB1, flags=direct, block_bytes=bb, lanes_per_gpu=lanes)
        regular = _regular_primaries(s)
        assert r1["files_trusted"] == 0 and r1["bytes_read"] == sum(st.st_size for st in regular.values())
        assert r1["bytes_h2d"] == r1["bytes_read"] + r1["bytes_verified"] and r1["files_verified"] == r1["files_read"]
        assert r1["src_recorded"] == sum(1 for st in regular.values() if st.st_size and st.st_nlink == 1), r1
        assert r1["src_recorded"] + r1["src_unrecorded"] == len(orc.read_table(sA1)["entries"])
        a1, b1 = orc.read_table(tA1), orc.read_table(tB1)
        assert a1["entries"] == b1["entries"] and (vm.table_hashes(tA1) == vm.table_hashes(tB1)).all()
        assert orc.read_table(sA1)["entries"] == a1["entries"] and (vm.table_hashes(sA1) == vm.table_hashes(tA1)).all()
        # pass 2 (paused) with pass 1's source table: what the tenant touched is read in full, the rest not at all
        _edit(s, bb)
        f = vm.F_PRUNE | verify | direct
        want = _paused_pass(vm, orc, root, s, sA1, dA, dB, tA1, tB1, f"2{k}", f, bb, lanes)
        assert all(want[rel] == 0 for rel in UNTOUCHED), want
        assert want[b"u/chmod.bin"] == 2 * bb and want[b"m/a.bin"] == 5 * bb + 123
        # pass 3 with a source table newer than the destination's: of a trusted file only the blocks that are not the
        # prior record's at the same index are read (a short tail block whose length changed included)
        _flip(s / "u" / "keep1.bin", bb + 3)
        with open(s / "u" / "keep2.bin", "ab") as fh:
            fh.write(b"x" * 100)
        os.truncate(s / "u" / "keep3.bin", 2 * bb + 9)
        _settle()
        sH = root / f"sH{k}.vmig"
        vm.hash_tree(s, sH, block_bytes=bb)
        want = _paused_pass(vm, orc, root, s, sH, dA, dB, root / f"tA2{k}.vmig", root / f"tB2{k}.vmig", f"3{k}", f, bb, lanes)
        assert want[b"u/keep0.bin"] == 0 and want[b"u/keep1.bin"] == bb, want
        assert want[b"u/keep2.bin"] == (3 * bb + 34 + 100) - 3 * bb and want[b"u/keep3.bin"] == 9, want


# ------------------------------------------------------------------------------------------ 2. a forged source table
def test_forged_src_table_fails_with_esrcchanged(vm, orc, shm_tmp):
    bb = 1 << 20
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    src.mkdir(), dst.mkdir()
    for i in range(4):
        (src / f"k{i}.bin").write_bytes(lm.data(200 + i, 3 * bb + i))
    _settle()
    t1, s1, t2 = shm_tmp / "t1.vmig", shm_tmp / "s1.vmig", shm_tmp / "t2.vmig"
    r = vm.migrate_layer(src, None, dst, None, t1, s1, flags=vm.F_VERIFY, block_bytes=bb)
    assert r["src_recorded"] == 4, r
    t = orc.read_table(s1)
    (first, ident), = [(f, i) for (rel, _, f), i in zip(t["entries"], t["identity"]) if rel == b"k2.bin"]
    assert ident[0] != 0
    raw = bytearray(s1.read_bytes())
    off = len(raw) - 8 * (len(t["hashes"]) - first - 1)
    raw[off] ^= 1                                                  # block 1 of k2.bin: no longer the prior's, so it is read
    s1.write_bytes(bytes(raw))
    before, dst_before, tables = src_state(src), src_state(dst), {p: p.read_bytes() for p in (t1, s1)}
    with pytest.raises(vm.VmigError) as ei:
        vm.migrate_layer(src, s1, dst, t1, t2, None, flags=vm.F_VERIFY | vm.F_PRUNE, block_bytes=bb)
    assert ei.value.code == vm.VMIG_ESRCCHANGED and "k2.bin block 1" in str(ei.value), ei.value
    assert not t2.exists()
    _no_tmp(t2)
    assert src_state(src) == before and src_state(dst) == dst_before            # the block's batch was not written
    assert all(p.read_bytes() == b for p, b in tables.items())


# ------------------------------------------------------------------------------------------ 3. a live writer in pass 1
def test_live_writer_during_pass1_is_read_in_pass2(vm, orc, shm_tmp):
    bb = 1 << 20
    src, dst, ref = shm_tmp / "src", shm_tmp / "dst", shm_tmp / "ref"
    src.mkdir(), dst.mkdir(), ref.mkdir()
    for i in range(8):
        (src / f"c{i}.bin").write_bytes(lm.data(300 + i, 24 * MiB + i))
    (src / "hot.bin").write_bytes(lm.data(399, 8 * MiB))
    _settle()
    stop = threading.Event()

    def tenant():
        k = 0
        while not stop.is_set():
            with open(src / "hot.bin", "r+b") as f:
                f.seek((k * 4099) % (8 * MiB - 64))
                f.write(lm.data(500 + k, 64))
            k += 1
            time.sleep(0.0002)
    th = threading.Thread(target=tenant)
    t1, s1, t2 = shm_tmp / "t1.vmig", shm_tmp / "s1.vmig", shm_tmp / "t2.vmig"
    th.start()
    try:
        vm.migrate_layer(src, None, dst, None, t1, s1, flags=vm.F_VERIFY, block_bytes=bb)
    finally:
        stop.set()
        th.join()
    _flip(src / "hot.bin", 12345)                                  # once more, after pass 1 returned
    r = vm.migrate_layer(src, s1, dst, t1, t2, None, flags=vm.F_VERIFY | vm.F_PRUNE, block_bytes=bb)
    assert r["bytes_read"] >= 8 * MiB and r["files_read"] >= 1, r
    orc.ref_copy(src, ref)
    assert orc.compare_trees(ref, dst) == []
    _, want = orc.block_table_of_tree(src, bb)
    assert (vm.table_hashes(t2) == want).all()


# ------------------------------------------------------------------------------------------ 4. cancel
def test_cancel_in_pass2_then_succeed(vm, orc, shm_tmp):
    bb = 4 << 20
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    src.mkdir(), dst.mkdir()
    for i in range(12):
        (src / f"f{i:02d}").write_bytes(lm.data(3 + i, 96 * MiB))
    _settle()
    t1, s1, t2 = shm_tmp / "t1.vmig", shm_tmp / "s1.vmig", shm_tmp / "t2.vmig"
    vm.migrate_layer(src, None, dst, None, t1, s1, block_bytes=bb)
    for i in range(12):                                            # every file changed: pass 2 reads all of them
        _flip(src / f"f{i:02d}", (i % 20) * bb + 3)
    tables = {p: p.read_bytes() for p in (t1, s1)}
    hit = False
    for _ in range(3):
        with vm.Ctl() as c:
            done = threading.Event()

            def canceller():
                while not done.is_set():
                    p = c.progress()
                    if p["phase_name"] == "DATA" and p["bytes_hashed"] >= p["bytes_total"] // 2 > 0:
                        c.cancel()
                        return
                    time.sleep(0.0002)
            th = threading.Thread(target=canceller)
            th.start()
            try:
                vm.migrate_layer(src, s1, dst, t1, t2, None, flags=vm.F_VERIFY | vm.F_PRUNE, block_bytes=bb, ctl=c)
                break                                              # the pass was too short to hit
            except vm.VmigError as e:
                assert e.code == vm.VMIG_ECANCELED and "cancelled in phase DATA" in str(e), e
                hit = True
            finally:
                done.set()
                th.join()
        assert not t2.exists()
        _no_tmp(t2)
        assert all(p.read_bytes() == b for p, b in tables.items())
        if hit:
            break
    assert hit, "a cancel half way through the data pass was not honoured"
    # the destination is half patched and the prior table no longer vouches for those files: they are read in full
    r = vm.migrate_layer(src, s1, dst, t1, t2, None, flags=vm.F_VERIFY | vm.F_PRUNE, block_bytes=bb)
    assert r["bytes_read"] > 0
    same_tree(orc, src, dst)
    _, want = orc.block_table_of_tree(src, bb)
    assert (vm.table_hashes(t2) == want).all()


# ------------------------------------------------------------------------------------------ 5. the hand-off mirror
def _handoff(vm):
    return importlib.import_module(vm.__name__ + ".handoff")


def test_handoff_from_layer_with_a_live_writer(vm, orc, shm_tmp):
    """HandoffCopyFromLayer with the tenant of tests/test_gpu.py::test_handoff_two_pass_with_a_live_writer: the paused
    pass reads only the files the tenant touched since the live pass began."""
    import numpy as np
    ho = _handoff(vm)
    old, new, ref = shm_tmp / "upper_old", shm_tmp / "upper_new", shm_tmp / "ref"
    old.mkdir(), new.mkdir(), ref.mkdir()
    sizes = {f"f{i:02d}.bin": (6 + i) * MiB + 17 * i for i in range(12)}
    for name, n in sizes.items():
        (old / name).write_bytes(orc.splitmix_bytes(700 + len(name) + n, n).tobytes())
    _settle()
    hot = ["f00.bin", "f01.bin", "f02.bin"]
    stop, paused = threading.Event(), threading.Event()

    def tenant():
        rng = np.random.default_rng(1)
        k = 0
        while not stop.is_set():
            name = hot[k % 3]
            with open(old / name, "r+b") as f:
                if k % 3 == 1:
                    f.seek(0, 2); f.write(rng.integers(0, 256, 7000, dtype=np.uint8).tobytes())       # append
                else:
                    f.seek(int(rng.integers(0, sizes[name] - 4096))); f.write(rng.integers(0, 256, 4096, dtype=np.uint8).tobytes())
            if k % 40 == 7:
                (old / f"new{k}.log").write_bytes(b"log line\n" * (k + 1))
            k += 1
            time.sleep(0.0005)
    th = threading.Thread(target=tenant)

    def pause(name):
        assert name == "rs-1"
        stop.set(); th.join(); paused.set()
        os.unlink(old / "f05.bin")
        os.rename(old / "f06.bin", old / "renamed06.bin")

    vm.set_resolver(container_upperdir=lambda n: str({"rs-1": old, "rs-2": new}[n]))
    ho.set_merges_root(shm_tmp)
    th.start()
    try:
        out = ho.HandoffCopyFromLayer("rs-1", "rs-2", pause, lambda n: pytest.fail("resume called: the final pass failed"))
    finally:
        stop.set()
        if th.is_alive():
            th.join()
        vm.set_resolver(None, None); ho.set_merges_root(None)
    assert paused.is_set() and out["pass1"] is not None and out["pass1_error"] is None, out
    p1, p2 = out["pass1"], out["pass2"]
    assert p1["files_verified"] == p1["files_read"] and p1["src_recorded"] > 0
    orc.ref_copy(old, ref)
    assert orc.compare_trees(ref, new) == []
    assert not (new / "f05.bin").exists() and not (new / "f06.bin").exists() and p2["pruned"] >= 2
    logs = [p.name for p in old.glob("new*.log")]
    touched = hot + logs + ["renamed06.bin"]
    assert 0 < p2["files_read"] <= len(touched), (p2, touched)
    assert p2["bytes_read"] <= sum((old / n).stat().st_size for n in touched), p2        # the cold files read 0 bytes
    assert p2["files_unread"] >= len(sizes) - len(hot) - 2
    vdir = shm_tmp / "merges" / "rs" / "rs-2"
    assert (vdir / "blocks.vmig").exists()
    assert sorted(os.listdir(vdir)) == ["blocks.vmig"]              # no .pass1 table (nor .tmp) left behind
    _, want = orc.block_table_of_tree(old)
    assert (vm.table_hashes(vdir / "blocks.vmig") == want).all()


def test_handoff_from_layer_pause_budget(vm, orc, shm_tmp):
    ho = _handoff(vm)
    old, new = shm_tmp / "upper_old", shm_tmp / "upper_new"
    old.mkdir(), new.mkdir()
    vm.datagen_files(old, 9, 4, 256 * MiB)
    calls, frozen = [], {}

    def pause(n):
        calls.append(("pause", n))
        for p in old.iterdir():                                    # the tenant wrote every file: pass 2 reads them all
            _flip(p, 7)
        frozen.update(src_state(old))

    vm.set_resolver(container_upperdir=lambda n: str({"rs-1": old, "rs-2": new}[n]))
    ho.set_merges_root(shm_tmp)
    try:
        with pytest.raises(vm.VmigError) as ei:
            ho.HandoffCopyFromLayer("rs-1", "rs-2", pause, lambda n: calls.append(("resume", n)), pauseBudget=0.005)
        assert ei.value.code == vm.VMIG_ECANCELED and getattr(ei.value, "pause_budget_exceeded", False), ei.value
        assert calls == [("pause", "rs-1"), ("resume", "rs-1")]
        assert src_state(old) == frozen
        vdir = shm_tmp / "merges" / "rs" / "rs-2"
        assert os.listdir(vdir) == []                              # no table, no .pass1 table, no .tmp
        calls.clear()
        out = ho.HandoffCopyFromLayer("rs-1", "rs-2", lambda n: calls.append(("pause", n)),
                                      lambda n: calls.append(("resume", n)), pauseBudget=0)
        assert calls == [("pause", "rs-1")] and out["pass1"] is not None
        ref = shm_tmp / "ref"
        ref.mkdir()
        orc.ref_copy(old, ref)
        assert orc.compare_trees(ref, new) == []
        _, want = orc.block_table_of_tree(old)
        assert (vm.table_hashes(vdir / "blocks.vmig") == want).all()
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
