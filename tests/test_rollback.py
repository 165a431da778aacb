"""vmig_rollback_layer on the GPU (-m gpu).  Every rollback of a layer L is held to a pruning restore of the same snapshot
into an identical copy L' (vmig_restore_tree, F_PRUNE) and to the snapshot itself (oracle.compare_trees), its out table to
the snapshot's table and to lstat of L, and its cost to vmig_compare_snapshot's counters taken on the same layer state:
the same files_read and bytes_read, and bytes_fetched equal to bytes_restore less the bytes compare counts for the second
and later paths of snapshot hard-link groups (restated here from lstat and oracle.hash_file)."""
import importlib
import os
import shutil
import stat
import threading
import time
from pathlib import Path

import numpy as np
import pytest

import _layer_model as lm
from conftest import make_rich_tree
from test_compare import _flip, _mutate, _setup

pytestmark = pytest.mark.gpu
MiB = 1 << 20
G4 = 1 << 32


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _walk(root) -> dict:
    root = os.fsencode(os.fspath(root))
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            out[os.path.relpath(p, root)] = os.lstat(p)
    return out


def restore_bytes(layer, snap, bb) -> tuple:
    """(bytes the rollback fetches, bytes compare counts for secondary paths of snapshot hard-link groups), by the rule
    of include/vmig.h: per snapshot regular path, the blocks the layer's regular file at the path lacks at the same index
    with the same (length, hash), or the whole file."""
    L, S = _walk(layer), _walk(snap)
    groups = {}
    for rel, s in S.items():
        if stat.S_ISREG(s.st_mode):
            groups.setdefault((s.st_dev, s.st_ino), []).append(rel)
    primary = {min(g) for g in groups.values()}
    fetch = second = 0
    for rel, s in S.items():
        if not stat.S_ISREG(s.st_mode):
            continue
        n = 0
        sh = _orc.hash_file(os.path.join(os.fsencode(os.fspath(snap)), rel), bb) if s.st_size else []
        l = L.get(rel)
        if l is None or not stat.S_ISREG(l.st_mode):
            n = s.st_size
        else:
            lh = _orc.hash_file(os.path.join(os.fsencode(os.fspath(layer)), rel), bb) if l.st_size else []
            for r in range(-(-s.st_size // bb)):
                slen = min(bb, s.st_size - r * bb)
                if r * bb >= l.st_size or min(bb, l.st_size - r * bb) != slen or int(lh[r]) != int(sh[r]):
                    n += slen
        if rel in primary:
            fetch += n
        else:
            second += n
    return fetch, second


_orc = None


@pytest.fixture(autouse=True)
def _oracle(orc):
    global _orc
    _orc = orc


def rollback_checked(vm, orc, root, layer, snap, table, bb, flags=0, layer_table=None, lanes=1, out=None):
    """Roll layer back, a copy of it by a pruning restore, and hold both, the out table and the cost to the oracle."""
    out = out or root / "out.vmig"
    copy = root / "copy"
    if copy.exists():
        shutil.rmtree(copy)
    lm.freeze(layer, copy)
    want_fetch, second = restore_bytes(layer, snap, bb)
    cmp = vm.compare_snapshot(layer, snap, table, None, layer_table, flags=flags & ~(vm.F_VERIFY | vm.F_PRUNE), block_bytes=bb,
                              lanes_per_gpu=lanes)
    r = vm.rollback_layer(layer, snap, table, out, layer_table, flags=flags, block_bytes=bb, lanes_per_gpu=lanes)
    vm.restore_tree(snap, table, copy, None, None, flags=vm.F_PRUNE | (flags & (vm.F_MTIME_NS | vm.F_NO_METADATA | vm.F_SKIP_HIDDEN_TOPDIRS)),
                    block_bytes=bb, lanes_per_gpu=lanes)
    ns = bool(flags & vm.F_MTIME_NS)
    assert orc.compare_trees(layer, copy, mtime_ns=ns) == []
    if not flags & vm.F_NO_METADATA:                                  # a store's inodes are also linked from other versions
        assert lm.diff_manifests(lm.tree_in_itself(orc, layer, ns), lm.tree_in_itself(orc, snap, ns)) == []
    # cost: compare's counters on the same state
    assert r["files_read"] == cmp["files_read"] and r["bytes_read"] == cmp["bytes_read"], (r, cmp)
    assert r["bytes_fetched"] == want_fetch and cmp["bytes_restore"] == want_fetch + second, (r, cmp, want_fetch, second)
    if not flags & vm.F_VERIFY:
        assert r["stats"]["bytes_h2d"] == r["bytes_read"] + r["bytes_fetched"]
    # the out table: the snapshot's paths, sizes and hashes, and L's identities as the call left them
    t, s = orc.read_table(out), orc.read_table(table)
    assert t["entries"] == s["entries"] and (vm.table_hashes(out) == vm.table_hashes(table)).all()
    for (rel, size, _f), (ino, ct) in zip(t["entries"], t["identity"]):
        if ino:
            st_ = os.lstat(os.path.join(os.fsencode(os.fspath(layer)), os.fsencode(rel) if isinstance(rel, str) else rel))
            assert (st_.st_ino, st_.st_ctime_ns, st_.st_size) == (ino, ct, size), rel
    # handed to a diff pass, it vouches for every file it records with an identity
    m = vm.migrate_tree(snap, layer, out, None, flags=flags & (vm.F_MTIME_NS | vm.F_NO_METADATA), block_bytes=bb)
    assert m["files_untrusted"] == 0
    return r, cmp


# ------------------------------------------------------------------------------------------ 1. a mutated layer
@pytest.mark.parametrize("bb,lanes", [(4 << 20, 1), (4 << 20, 3), (65536, 1), (65536, 3), ((1 << 20) + 4096, 1), ((1 << 20) + 4096, 3)])
def test_mutated_layer_matches_restore(vm, orc, shm_tmp, bb, lanes):
    src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, lanes)
    _mutate(layer, bb)
    r, _ = rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb, lanes=lanes)
    assert r["files_patched"] and r["files_rebuilt"] and r["files_created"] and r["files_kept"], r
    # the same mutations under the metadata flags, and VMIG_F_VERIFY
    for flags in (vm.F_MTIME_NS, vm.F_VERIFY | vm.F_DIRECT_IO):
        _mutate(layer, bb)
        rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb, flags=flags, lanes=lanes)


def test_layer_group_over_separate_snapshot_files(vm, orc, shm_tmp):
    """One layer inode at three paths the snapshot holds as three files: each path is rebuilt in turn, and the call's own
    unlinks of the group's earlier paths do not fail the re-check of the later ones (one of them takes a fetched block,
    so it is rebuilt on a pipeline writer)."""
    bb = 65536
    src, snap, layer = shm_tmp / "src", shm_tmp / "snap", shm_tmp / "layer"
    (src / "g").mkdir(parents=True)
    body = lm.data(5, 3 * bb + 17)
    for n in ("a", "b", "c"):
        (src / "g" / n).write_bytes(body if n != "c" else body[:bb] + lm.data(6, bb) + body[2 * bb:])
    (src / "other").write_bytes(lm.data(7, 2 * bb))
    snap.mkdir()
    layer.mkdir()
    vm.snapshot_tree(src, snap, None, None, shm_tmp / "snap.vmig", block_bytes=bb)
    vm.restore_tree(snap, shm_tmp / "snap.vmig", layer, None, shm_tmp / "layer.vmig", block_bytes=bb)
    for n in ("b", "c"):
        os.unlink(layer / "g" / n)
        os.link(layer / "g" / "a", layer / "g" / n)
    time.sleep(0.02)
    for lanes in (1, 3):
        r, _ = rollback_checked(vm, orc, shm_tmp, layer, snap, shm_tmp / "snap.vmig", bb, lanes=lanes)
        assert r["files_rebuilt"] == 3 and r["blocks_fetched"] == 1 and r["bytes_copied"] == 3 * (3 * bb + 17) - bb, r
        assert len({os.stat(layer / "g" / n).st_ino for n in ("a", "b", "c")}) == 3
        for n in ("b", "c"):                                          # the group again, for the next lane count
            os.unlink(layer / "g" / n)
            os.link(layer / "g" / "a", layer / "g" / n)
        time.sleep(0.02)


# ------------------------------------------------------------------------------------------ 2. the layer's trust
def test_layer_table_trusted_none_and_stale(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, hardlinks=False)
    _flip(layer / "big.bin", 3 * bb + 1, keep_mtime=False)
    _flip(layer / "mb" / "mid", bb + 5, keep_mtime=True)
    r, cmp = rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb, layer_table=lt, out=lt)    # carried forward in place
    assert r["files_trusted"] > 0 and r["files_read"] == 2 and r["files_patched"] == 2 and r["bytes_fetched"] == 2 * bb, r
    _flip(layer / "exact.bin", 7, keep_mtime=False)                   # its own table again: only the edit is read
    r, _ = rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb, layer_table=lt)
    assert r["files_read"] == 1 and r["bytes_fetched"] == min(bb, (layer / "exact.bin").stat().st_size)
    stale = shm_tmp / "stale.vmig"
    shutil.copy(lt, stale)
    _flip(layer / "mb" / "first", 0, keep_mtime=False)               # a table older than the layer: untrusted where stale
    os.truncate(layer / "mb" / "shrink", bb + 10)
    (layer / "newfile").write_bytes(b"new")
    rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb, layer_table=stale)
    _flip(layer / "big.bin", 5)
    r, _ = rollback_checked(vm, orc, shm_tmp, layer, snap, t, bb)     # no table: every file the snapshot has is read
    assert r["files_trusted"] == 0 and r["files_read"] > 0


# ------------------------------------------------------------------------------------------ 3. nothing to do
def test_identical_layer_reads_and_writes_nothing(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, hardlinks=False)
    before = {rel: (s.st_ino, s.st_ctime_ns) for rel, s in _walk(layer).items() if stat.S_ISREG(s.st_mode)}
    r = vm.rollback_layer(layer, snap, t, lt, lt, block_bytes=bb)
    assert r["stats"]["bytes_h2d"] == 0 and r["stats"]["bytes_written"] == 0 and r["bytes_read"] == 0 and r["bytes_fetched"] == 0
    assert r["files_kept"] > 0 and r["files_patched"] + r["files_rebuilt"] + r["files_created"] == 0, r
    after = {rel: (s.st_ino, s.st_ctime_ns) for rel, s in _walk(layer).items() if stat.S_ISREG(s.st_mode)}
    assert after == before                                            # no regular file's ctime moved: still trusted
    assert orc.compare_trees(layer, snap) == []


# ------------------------------------------------------------------------------------------ 4. the store is only read
def test_store_untouched_and_never_shared(vm, orc, shm_tmp):
    bb, n = 65536, 3
    src = shm_tmp / "src"
    lm.build_layer(src, orc, bb, make_rich_tree)
    ops = [[]] + lm.script(33, n, bb)
    V = []
    for k in range(n + 1):
        lm.apply(src, ops[k])
        d, tab = shm_tmp / f"v{k}", shm_tmp / f"v{k}.vmig"
        d.mkdir()
        base = V[-1] if V else (None, None)
        vm.snapshot_tree(src, d, base[0], base[1], tab, block_bytes=bb)
        V.append((d, tab))
    store = lambda: {(d, rel): (s.st_ino, s.st_mode, s.st_mtime_ns, s.st_ctime_ns,
                                orc.hash_file(os.path.join(os.fsencode(os.fspath(d)), rel), bb).tobytes() if stat.S_ISREG(s.st_mode) else b"")
                     for d, _t in V for rel, s in _walk(d).items()}
    store_inodes = lambda: {(s.st_dev, s.st_ino) for d, _t in V for s in _walk(d).values() if stat.S_ISREG(s.st_mode)}
    for j, k in ((0, n), (n, 0), (1, 2)):
        layer = shm_tmp / f"layer_{j}_{k}"
        subprocess_cp_al(V[k][0], layer)                             # every layer file a hard link into version k
        (shm_tmp / "outside").mkdir(exist_ok=True)
        victim = next(rel for rel, s in sorted(_walk(layer).items()) if stat.S_ISREG(s.st_mode) and s.st_size)
        os.unlink(layer / os.fsdecode(victim))                        # one file of its own, also linked outside the tree
        shutil.copy2(V[k][0] / os.fsdecode(victim), layer / os.fsdecode(victim))
        _flip(layer / os.fsdecode(victim), 0)
        os.link(layer / os.fsdecode(victim), shm_tmp / "outside" / f"{j}{k}")
        held = open(shm_tmp / "outside" / f"{j}{k}", "rb").read()
        linked = {(s.st_dev, s.st_ino) for s in _walk(layer).values() if stat.S_ISREG(s.st_mode)}
        before = store()
        rollback_checked(vm, orc, shm_tmp, layer, V[j][0], V[j][1], bb)
        after = store()
        assert before.keys() == after.keys()
        for key, (ino, mode, mt, ct, h) in before.items():
            a = after[key]
            assert (a[0], a[1], a[2], a[4]) == (ino, mode, mt, h), key
            # an unlink moves the ctime of the inode it unlinks: only inodes the layer held a link to may show it
            assert a[3] == ct or (os.lstat(os.path.join(os.fsencode(os.fspath(key[0])), key[1])).st_dev, ino) in linked, key
        assert not {(s.st_dev, s.st_ino) for s in _walk(layer).values() if stat.S_ISREG(s.st_mode)} & store_inodes()
        assert open(shm_tmp / "outside" / f"{j}{k}", "rb").read() == held


def subprocess_cp_al(src, dst):
    import subprocess
    subprocess.run(["cp", "-a", "-l", os.fspath(src), os.fspath(dst)], check=True)


# ------------------------------------------------------------------------------------------ 5. a damaged snapshot
def test_damaged_snapshot_block(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, hardlinks=False)
    _flip(snap / "mb" / "mid", bb + 9)                                 # rotted, and the layer holds the good block
    r = vm.rollback_layer(layer, snap, t, None, lt, block_bytes=bb)
    assert r["bytes_fetched"] == 0
    t_rec = {e[0] if isinstance(e[0], str) else os.fsdecode(e[0]): e for e in orc.read_table(t)["entries"]}
    hs = vm.table_hashes(t)
    rel, size, first = t_rec["mb/mid"]
    assert (orc.hash_file(layer / "mb" / "mid", bb) == hs[first:first + -(-size // bb)]).all()
    _flip(snap / "mb" / "first", 3)                                    # rotted, and the layer needs that block
    _flip(layer / "mb" / "first", 3 + 1)
    good = (layer / "mb" / "first").read_bytes()[:bb]
    bad = (snap / "mb" / "first").read_bytes()[:bb]
    with pytest.raises(vm.VmigError) as ei:
        vm.rollback_layer(layer, snap, t, shm_tmp / "o.vmig", lt, block_bytes=bb)
    assert ei.value.code == vm.VMIG_ECORRUPT and "mb/first" in str(ei.value), ei.value
    assert (layer / "mb" / "first").read_bytes()[:bb] != bad and (layer / "mb" / "first").read_bytes()[:bb] == good
    assert not any(n.startswith("o.vmig") for n in os.listdir(shm_tmp))


# ------------------------------------------------------------------------------------------ 6. past 4 GiB
def test_changed_block_past_4gib(vm, orc, shm_tmp):
    st = os.statvfs(shm_tmp)
    if st.f_bavail * st.f_frsize < (7 << 30):
        pytest.skip("needs 7 GiB free in the test directory for a snapshot past 4 GiB")
    bb, size = 4 << 20, G4 + 9 * MiB + 777
    src, snap, layer = shm_tmp / "src", shm_tmp / "snap", shm_tmp / "layer"
    for d in (src, snap, layer):
        d.mkdir()
    islands = [(0, 2 * MiB), (G4 - MiB, 3 * MiB), (size - 5 * MiB, 5 * MiB)]

    def sparse(p, seed):
        with open(p, "wb") as f:
            f.truncate(size)
            for i, (off, n) in enumerate(islands):
                f.seek(off)
                f.write(lm.data(seed + i, n))
    sparse(src / "big", 1)
    vm.snapshot_tree(src, snap, None, None, shm_tmp / "snap.vmig", block_bytes=bb)
    shutil.rmtree(src)
    sparse(layer / "big", 1)
    os.utime(layer / "big", ns=(os.stat(snap / "big").st_atime_ns, os.stat(snap / "big").st_mtime_ns))
    os.chmod(layer / "big", stat.S_IMODE(os.stat(snap / "big").st_mode))
    off = G4 + bb + 12345                                             # a changed full block past 2^32
    with open(layer / "big", "r+b") as f:
        f.seek(off)
        f.write(b"\xAB" * 100)
    ino = os.stat(layer / "big").st_ino
    r = vm.rollback_layer(layer, snap, shm_tmp / "snap.vmig", None, None, block_bytes=bb)
    assert r["files_patched"] == 1 and r["blocks_fetched"] == 1 and r["bytes_fetched"] == bb and os.stat(layer / "big").st_ino == ino
    with open(layer / "big", "rb") as a, open(snap / "big", "rb") as b:
        a.seek(off - 12345)
        b.seek(off - 12345)
        assert a.read(bb) == b.read(bb)
    assert (orc.hash_file(layer / "big", bb) == vm.table_hashes(shm_tmp / "snap.vmig")).all()


# ------------------------------------------------------------------------------------------ 7. cancel and phases
def test_cancel_in_each_phase_then_succeed(vm, orc, shm_tmp):
    bb = 4 << 20
    src, snap, layer = shm_tmp / "src", shm_tmp / "snap", shm_tmp / "layer"
    src.mkdir()
    for i in range(12):
        (src / f"f{i:02d}").write_bytes(lm.data(3 + i, 96 * MiB))
    (src / "d").mkdir()
    for i in range(3000):
        (src / "d" / f"s{i}").write_bytes(b"s%d" % i)
    snap.mkdir()
    vm.snapshot_tree(src, snap, None, None, shm_tmp / "snap.vmig", block_bytes=bb)
    order = ["IDLE", "WALK", "PRUNE", "DATA", "META", "VERIFY", "TABLE", "DONE"]

    def mutate():
        for i in range(12):
            _flip(layer / f"f{i:02d}", (i % 20) * bb + 3)
        (layer / "extra").write_bytes(b"pruned")
    lm.freeze(src, layer)
    mutate()
    for target in ("DATA", "WALK", "PRUNE", "META", "TABLE"):
        with vm.Ctl() as c:
            returned = threading.Event()

            def canceller():
                while not returned.is_set():
                    p = c.progress()
                    if p["phase_name"] == target and (target != "DATA" or p["bytes_hashed"] >= p["bytes_total"] // 2):
                        c.cancel()
                        return
                    time.sleep(0.0002)
            th = threading.Thread(target=canceller)
            th.start()
            try:
                vm.rollback_layer(layer, snap, shm_tmp / "snap.vmig", shm_tmp / "out.vmig", None, flags=vm.F_VERIFY, block_bytes=bb, ctl=c)
                assert target != "DATA", "a cancel half way through the data pass was not honoured"
                mutate()                                              # the phase was too short to hit: start over
            except vm.VmigError as e:
                stopped = str(e).split("cancelled in phase ")[1].split(":")[0]
                assert e.code == vm.VMIG_ECANCELED and order.index(stopped) >= order.index(target), e
                assert not any(n.startswith("out.vmig") for n in os.listdir(shm_tmp))
            finally:
                returned.set()
                th.join()
    with vm.Ctl() as c:
        seen, done, prog = [], threading.Event(), []

        def watch():
            while not done.is_set():
                p = c.progress()
                prog.append((p["bytes_total"], p["bytes_hashed"], p["bytes_written"]))
                if not seen or seen[-1] != p["phase_name"]:
                    seen.append(p["phase_name"])
                time.sleep(0.0002)
        th = threading.Thread(target=watch)
        th.start()
        try:
            r = vm.rollback_layer(layer, snap, shm_tmp / "snap.vmig", shm_tmp / "out.vmig", None, flags=vm.F_VERIFY, block_bytes=bb, ctl=c)
        finally:
            done.set()
            th.join()
        final = c.progress()
        seen.append(final["phase_name"])
    assert [order.index(p) for p in seen] == sorted(order.index(p) for p in seen) and seen[-1] == "DONE", seen
    for i in range(3):
        assert all(a[i] <= b[i] for a, b in zip(prog, prog[1:])), i
    assert orc.compare_trees(layer, snap) == []
    assert final["bytes_total"] == r["stats"]["bytes_total"] == r["bytes_read"] + r["bytes_fetched"]
    assert final["bytes_written"] == r["stats"]["bytes_written"] == r["bytes_fetched"]


# ------------------------------------------------------------------------------------------ 8. alongside other calls
def test_rollback_alongside_a_migration_and_a_snapshot(vm, orc, shm_tmp):
    bb = 1 << 20
    src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    _mutate(layer, bb)
    copy = shm_tmp / "copy"
    lm.freeze(layer, copy)
    big = shm_tmp / "big"
    big.mkdir()
    for i in range(6):
        (big / f"f{i}").write_bytes(lm.data(80 + i, 48 * MiB + i))
    (shm_tmp / "mig").mkdir()
    (shm_tmp / "inc").mkdir()
    (src / "edited").write_bytes(b"for the increment")
    errs, out = [], {}

    def run(name, fn):
        try:
            out[name] = fn()
        except Exception as e:                       # noqa: BLE001 -- reported below
            errs.append((name, e))
    calls = {
        "rollback": lambda: vm.rollback_layer(layer, snap, t, shm_tmp / "out.vmig", None, block_bytes=bb, lanes_per_gpu=2),
        "migrate": lambda: vm.migrate_tree(big, shm_tmp / "mig", block_bytes=bb),
        "snapshot": lambda: vm.snapshot_tree(src, shm_tmp / "inc", snap, t, shm_tmp / "inc.vmig", block_bytes=bb),
    }
    ths = [threading.Thread(target=run, args=kv) for kv in calls.items()]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errs, errs
    vm.restore_tree(snap, t, copy, None, None, flags=vm.F_PRUNE, block_bytes=bb)
    assert orc.compare_trees(layer, copy) == []
    assert lm.diff_manifests(lm.tree_in_itself(orc, layer), lm.tree_in_itself(orc, snap)) == []   # inc now links into snap
    assert orc.compare_trees(big, shm_tmp / "mig") == []
    full = shm_tmp / "full"
    full.mkdir()
    vm.snapshot_tree(src, full, None, None, shm_tmp / "full.vmig", block_bytes=bb)
    assert lm.diff_manifests(lm.tree_in_itself(orc, full), lm.tree_in_itself(orc, shm_tmp / "inc")) == []


# ------------------------------------------------------------------------------------------ 9. the hand-off mirror
def test_rollback_in_place_after_a_handoff(vm, orc, shm_tmp):
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {n: shm_tmp / f"upper_{n}" for n in ("rs-1", "rs-2", "rs-3")}
    ups["rs-1"].mkdir()
    ups["rs-3"].mkdir()
    make_rich_tree(ups["rs-1"], orc)
    os.unlink(ups["rs-1"] / "sub" / "hard1")
    os.unlink(ups["rs-1"] / "a_hard2")
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersion("rs-1")
        lm.freeze(ups["rs-1"], ups["rs-2"])
        st1 = os.stat(ups["rs-1"])
        os.chmod(ups["rs-2"], stat.S_IMODE(st1.st_mode))
        os.utime(ups["rs-2"], ns=(st1.st_atime_ns, st1.st_mtime_ns))
        ho.HandoffCopy("rs-2", "rs-3", pause=lambda n: None, resume=lambda n: None)
        _flip(ups["rs-3"] / "exact.bin", 5, keep_mtime=True)          # the tenant's edit, and a new file
        (ups["rs-3"] / "new.txt").write_bytes(b"tenant")
        cmp = ho.CompareWithVersion("rs-1", "rs-3", shm_tmp / "cmp.txt")
        r = ho.RollbackInPlace("rs-1", "rs-3")
        data, table = ho.snapshotPaths("rs-1")
        assert r["bytes_fetched"] == cmp["bytes_restore"] == min(4 << 20, (data / "exact.bin").stat().st_size)
        assert r["files_read"] == cmp["files_read"] == 1 and r["files_trusted"] > 0
        assert orc.compare_trees(ups["rs-3"], data) == []
        r = ho.RollbackInPlace("rs-1", "rs-3")                        # its own table, carried forward: nothing to do
        assert r["bytes_read"] == 0 and r["bytes_fetched"] == 0 and r["files_kept"] > 0
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
