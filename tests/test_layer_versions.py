"""The layer calls chained as production chains them, on the GPU (-m gpu): one live layer through nine versions.

Every layer call trusts records an earlier call wrote: the hand-off's migration writes the layer's table, a rollback
rewrites it in place, a layer snapshot links unchanged files to base inodes (their ctimes move), a retire unlinks old
versions and re-stamps the kept records, and compare and snapshot_layer take whatever records are left.  A wrong record
does not show in the call that wrote it, only later, as a version that silently lacks a change.  So each version here is
taken twice from the same layer at the same moment: store A by vmig_snapshot_layer through the layer's table, store B
by vmig_snapshot_tree, which trusts no layer record, and both are held to a frozen copy of the layer and to the
oracle's table.  Every expected value is computed before its call, from the oracle, lstat and the tables as written.
Nothing waits between a call and the next edit: the next version's edits start the moment a call returns."""
import importlib
import json
import os
import shutil
import stat
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import _layer_model as L
import test_compare as TC
import test_rollback as TR
import test_snapshot_layer as TS
from conftest import make_rich_tree
from test_compare import _oracle_modules  # noqa: F401 -- autouse: sets the globals test_compare.expected reads
from test_rollback import _oracle  # noqa: F401 -- autouse: sets the global test_rollback.restore_bytes reads
from test_versions import _frozen, _regular_inodes

pytestmark = pytest.mark.gpu
N = 8
RETIRE_AT, RETIRED, KEPT_AT_RETIRE = 5, (1, 2, 3), [0, 4, 5]


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


# ------------------------------------------------------------------------------------------------ oracle helpers
def rollback_read(orc, layer, snap, layer_table, unlink_moves_ctime: bool = True) -> tuple:
    """(files_read, bytes_read, extra) of vmig_rollback_layer(layer, layer_table, snap) on the layer as it stands, by
    include/vmig.h: vmig_compare_snapshot's read plan, taken after the prune.  extra: {(st_dev, st_ino): size} of the
    documented exception -- inodes the table vouches for at a path both trees have, that lose another path to the prune
    (their ctime moves, so the rollback reads them), and that the compare reads under no other path.  files_read and
    bytes_read less extra are what a compare of the same state reads.  Where an unlink does not move the ctime of the
    inode it unlinks (unlink_moves_ctime False: some sandboxed kernels), there is no exception."""
    Lw, Sw = TC._walk(layer), TC._walk(snap)
    isdir = lambda st: stat.S_ISDIR(st.st_mode)

    def pruned(rel: bytes) -> bool:
        parts = rel.split(b"/")
        for i in range(1, len(parts)):
            d = b"/".join(parts[:i])
            if d not in Sw or not isdir(Sw[d]):
                return True
        return rel not in Sw or isdir(Sw[rel]) != isdir(Lw[rel])
    gone = {rel for rel in Lw if rel != b"." and pruned(rel)}
    lost_link = {(st.st_dev, st.st_ino) for rel, st in Lw.items() if rel in gone and stat.S_ISREG(st.st_mode)}
    t = orc.read_table(layer_table) if layer_table else {"entries": [], "identity": []}
    rec = {rel: (size, ino, ct) for (rel, size, _first), (ino, ct) in zip(t["entries"], t["identity"])}
    read, trusted_lost = {}, {}
    for rel, l in Lw.items():
        s = Sw.get(rel)
        if rel in gone or not stat.S_ISREG(l.st_mode) or s is None or not stat.S_ISREG(s.st_mode) or not l.st_size or not s.st_size:
            continue
        key = (l.st_dev, l.st_ino)
        if key == (s.st_dev, s.st_ino) and l.st_size == s.st_size:
            continue                                                   # shared with the snapshot: not read
        r = rec.get(rel)
        if r and r[1] and r == (l.st_size, l.st_ino, l.st_ctime_ns):
            if key in lost_link and unlink_moves_ctime:
                trusted_lost[key] = l.st_size
            continue
        read[key] = l.st_size
    extra = {key: size for key, size in trusted_lost.items() if key not in read}
    read.update(extra)
    return len(read), sum(read.values()), extra


def _unlink_moves_ctime(root: Path) -> bool:
    """Whether removing one link of an inode on root's filesystem moves the inode's ctime (Linux does)."""
    a, b = root / "probe_a", root / "probe_b"
    a.write_bytes(b"probe")
    os.link(a, b)
    before = os.lstat(a).st_ctime_ns
    time.sleep(0.05)                       # past the timer tick of the link, on any kernel
    os.unlink(b)
    moved = os.lstat(a).st_ctime_ns != before
    os.unlink(a)
    return moved


def _same_as_frozen(orc, frozen: Path, tree: Path, ns: bool, ctx):
    assert L.diff_manifests(_frozen(orc, frozen, ns), L.tree_in_itself(orc, tree, ns)) == [], ctx


def _table_is(orc, table: Path, want, ctx):
    got = orc.read_table(table)
    assert got["entries"] == want[0] and np.array_equal(got["hashes"], want[1]), ctx


def _identities_are_lstat(orc, table: Path, root: Path, ctx):
    t = orc.read_table(table)
    for (rel, size, _f), (ino, ct) in zip(t["entries"], t["identity"]):
        if ino:
            st = os.lstat(os.path.join(os.fsencode(os.fspath(root)), rel))
            assert (st.st_ino, st.st_ctime_ns, st.st_size) == (ino, ct, size), (ctx, rel)


def _regular_keys(root: Path) -> set:
    return set(_regular_inodes(root))


def _first_path(root: Path, key) -> bytes:
    """The bytewise-first path of the inode key in the tree: its hard-link group's primary."""
    r = os.fsencode(os.fspath(root))
    return min(os.path.relpath(os.path.join(dp, n), r) for dp, _d, fns in os.walk(r) for n in fns
               if (lambda st: (st.st_dev, st.st_ino))(os.lstat(os.path.join(dp, n))) == key)


def _group_inodes(root: Path) -> set:
    """(st_dev, st_ino) of the non-empty regular files that have more than one path in the tree."""
    paths = {}
    for dp, _d, fns in os.walk(os.fsencode(os.fspath(root))):
        for n in fns:
            st = os.lstat(os.path.join(dp, n))
            if stat.S_ISREG(st.st_mode) and st.st_size:
                paths[(st.st_dev, st.st_ino)] = paths.get((st.st_dev, st.st_ino), 0) + 1
    return {key for key, n in paths.items() if n > 1}


def _flip_at(p, off: int, xor: int = 0x5A):
    with open(p, "r+b") as f:
        f.seek(off)
        c = f.read(1)
        f.seek(off)
        f.write(bytes([c[0] ^ xor]))


CLOCK_REALTIME_COARSE = 5                # <linux/time.h>; the time module does not name it
TICK_NS = int(time.clock_getres(CLOCK_REALTIME_COARSE) * 1e9)
ROT = 0x3C                               # the damage: an XOR no edit of the script (0x5A, 0xA5) makes


def _edit_in_the_record_tick(orc, layer: Path, table: Path, rng, ctx) -> bytes:
    """Right after a call wrote `table`: a same-size edit of a single-link file it vouches for.  Its ctime must move
    whatever the kernel's timestamp granularity, or the next call would take the record's stale hashes."""
    t = orc.read_table(table)
    cands = []
    for (rel, size, _f), (ino, ct) in zip(t["entries"], t["identity"]):
        if not ino or not size:
            continue
        st = os.lstat(os.path.join(os.fsencode(os.fspath(layer)), rel))
        if (st.st_ino, st.st_ctime_ns, st.st_nlink) == (ino, ct, 1) and st.st_mode & 0o200:
            cands.append((rel, size, ct))
    assert cands, ctx
    rel, size, ct = cands[int(rng.integers(len(cands)))]
    p = os.path.join(os.fsencode(os.fspath(layer)), rel)
    _flip_at(p, size // 2)
    after = os.lstat(p).st_ctime_ns
    print(f"record tick: {ctx}: {rel!r} recorded ctime {ct}, ctime after the edit {after} "
          f"(+{after - ct} ns; coarse clock tick {TICK_NS} ns)")
    assert after != ct, (ctx, rel, ct)
    return rel


# ------------------------------------------------------------------------------------------------ the chain
CASES = [(31, 65536, 1, (), False), (32, 65536, 3, ("F_VERIFY",), False), (33, 4 << 20, 1, ("F_MTIME_NS",), False),
         (34, (1 << 20) + 4096, 3, ("F_VERIFY", "F_DIRECT_IO"), True), (35, 4096, 1, (), False)]


@pytest.mark.parametrize("seed,bb,lanes,flag_names,disk", CASES, ids=[f"seed{c[0]}" for c in CASES])
def test_layer_calls_through_nine_versions(vm, orc, shm_tmp, tmp_path, seed, bb, lanes, flag_names, disk):
    root = tmp_path if disk else shm_tmp
    F = 0
    for n in flag_names:
        F |= getattr(vm, n)
    ns = bool(F & vm.F_MTIME_NS)
    f_cmp, f_store = F & (vm.F_DIRECT_IO | vm.F_MTIME_NS), F & vm.F_DIRECT_IO
    kw = dict(block_bytes=bb, lanes_per_gpu=lanes)
    tag = f"seed {seed} bb {bb} lanes {lanes} flags {flag_names} {'disk' if disk else 'shm'}"
    ops = [[]] + L.script(seed, N, bb)
    rng = np.random.default_rng(seed + 1000)
    detours = {int(rng.integers(1, 4)), int(rng.integers(4, 6)), int(rng.integers(6, N))}
    src, layer, LT, report = root / "src", root / "layer", root / "LT.vmig", root / "cmp.txt"
    A, B = (lambda k: root / f"A{k}"), (lambda k: root / f"B{k}")
    TA, TB = (lambda k: root / f"A{k}.vmig"), (lambda k: root / f"B{k}.vmig")
    frozen = lambda k: root / f"frozen{k}"
    state, O, kept = {}, {}, []
    unlink_moves_ctime = _unlink_moves_ctime(root)

    def remember(k):
        for d in (A(k), B(k)):
            state[d] = L.tree_in_itself(orc, d, mtime_ns=True)
        kept.append(k)

    def stores_unchanged(ctx):
        for d, man in state.items():
            assert L.diff_manifests(man, L.tree_in_itself(orc, d, mtime_ns=True)) == [], (ctx, d.name)

    store_inodes = lambda: set().union(*(_regular_keys(d) for d in state))

    def compare_checked(snap, table, ctx):
        want, c = TC.expected(layer, snap, bb, f_cmp, LT)
        r = vm.compare_snapshot(layer, snap, table, report, LT, flags=f_cmp, **kw)
        assert report.read_bytes() == want, (ctx, report.read_bytes()[:2000], want[:2000])
        assert {x: r[x] for x in TC.COUNTERS} == c, (ctx, r, c)
        return r

    def rollback_checked(j, target_frozen, ctx):
        """Roll the layer back to A_j in place with LT as its table and its out table, held to a pruning restore of a
        copy, to the frozen version, to the compare of the same state and to the snapshot's table."""
        cmp = compare_checked(A(j), TA(j), ctx + " compare before")
        want_fetch, second = TR.restore_bytes(layer, A(j), bb)
        want_files, want_bytes, extra = rollback_read(orc, layer, A(j), LT, unlink_moves_ctime)
        assert (want_files - len(extra), want_bytes - sum(extra.values())) == (cmp["files_read"], cmp["bytes_read"]), ctx
        assert cmp["bytes_restore"] == want_fetch + second, (ctx, cmp, want_fetch, second)
        copy = root / "copy"
        shutil.rmtree(copy, ignore_errors=True)
        L.freeze(layer, copy)
        r = vm.rollback_layer(layer, A(j), TA(j), LT, LT, flags=F, **kw)
        vm.restore_tree(A(j), TA(j), copy, None, None, flags=vm.F_PRUNE | (F & vm.F_MTIME_NS), **kw)
        assert orc.compare_trees(layer, copy, mtime_ns=ns) == [], ctx
        _same_as_frozen(orc, target_frozen, layer, ns, ctx)
        assert r["bytes_fetched"] == want_fetch, (ctx, r, want_fetch)
        assert (r["files_read"], r["bytes_read"]) == (want_files, want_bytes), (ctx, r, want_files, want_bytes, extra)
        if not F & vm.F_VERIFY:
            assert r["stats"]["bytes_h2d"] == r["bytes_read"] + r["bytes_fetched"], (ctx, r)
        _table_is(orc, LT, (orc.read_table(TA(j))["entries"], orc.read_table(TA(j))["hashes"]), ctx)
        _identities_are_lstat(orc, LT, layer, ctx)
        assert not _regular_keys(layer) & store_inodes(), ctx
        stores_unchanged(ctx)
        # the table the rollback wrote vouches for every file it records: only hard-link groups are read again
        r2 = compare_checked(A(j), TA(j), ctx + " compare after")
        groups = _group_inodes(layer)
        assert r2["files_read"] == len(groups) and report.read_bytes() == b"", (ctx, r2)
        return r, extra

    # ---- version 0: the hand-off's migration writes the layer and its table; the first versions are full snapshots
    L.build_layer(src, orc, bb, make_rich_tree)
    layer.mkdir()
    vm.migrate_tree(src, layer, None, LT, flags=vm.F_PRUNE | vm.F_VERIFY | (F & (vm.F_DIRECT_IO | vm.F_MTIME_NS)), **kw)
    L.freeze(layer, frozen(0))
    O[0] = orc.block_table_of_tree(layer, bb)
    for S, T in ((A, TA), (B, TB)):
        S(0).mkdir()
        vm.snapshot_tree(layer, S(0), None, None, T(0), flags=F, **kw)
        _same_as_frozen(orc, frozen(0), S(0), ns, f"{tag} version 0")
        _table_is(orc, T(0), O[0], f"{tag} version 0")
    remember(0)
    extras = 0

    for k in range(1, N + 1):
        ctx = f"{tag} version {k}: {json.dumps(ops[k])}"
        L.apply(layer, ops[k])
        L.freeze(layer, frozen(k))
        O[k] = orc.block_table_of_tree(layer, bb)

        # ---- the version, twice: through the layer's table into A, by a full read into B
        base = max(kept)
        s = SimpleNamespace(base=A(base), bt=TA(base), layer=layer, lt=LT, dst=A(k))
        want_trusted, want_read = TS.expected_read(vm, orc, s, bb)
        before = TS.layer_state(layer)
        A(k).mkdir()
        B(k).mkdir()
        rb = vm.snapshot_tree(layer, B(k), B(base), TB(base), TB(k), flags=F, **kw)
        ra = vm.snapshot_layer(layer, A(k), A(base), TA(base), TA(k), LT, flags=F, **kw)
        assert TS.layer_state(layer) == before, ctx
        assert (ra["files_trusted"], ra["bytes_read"]) == (want_trusted, want_read), (ctx, ra, want_trusted, want_read)
        verify_bytes = TS.written_bytes(s) if F & vm.F_VERIFY else 0
        assert ra["bytes_h2d"] == ra["bytes_read"] + verify_bytes and ra["bytes_total"] == ra["bytes_read"], (ctx, ra)
        _same_as_frozen(orc, frozen(k), A(k), ns, ctx)
        _same_as_frozen(orc, frozen(k), B(k), ns, ctx)
        _table_is(orc, TA(k), O[k], ctx)
        _table_is(orc, TB(k), O[k], ctx)
        assert TS.links(A(k), A(base)) == TS.links(B(k), B(base)), ctx
        assert {x: ra[x] for x in TS.SHARED} == {x: rb[x] for x in TS.SHARED}, (ctx, ra, rb)
        assert ra["files_base_untrusted"] == 0, (ctx, ra)
        stores_unchanged(ctx)
        remember(k)

        # ---- what changed since the version was taken: nothing, at the cost of the files LT no longer vouches for
        compare_checked(A(k), TA(k), ctx + " compare")

        # ---- a detour to an earlier version and back, in place, LT rewritten by each rollback
        if k in detours:
            j = [v for v in kept if v < k][int(rng.integers(len([v for v in kept if v < k])))]
            _, ex = rollback_checked(j, frozen(j), f"{ctx} rollback to {j}")
            extras += len(ex)
            _, ex = rollback_checked(k, frozen(k), f"{ctx} roll forward from {j}")
            extras += len(ex)
            if k < N:               # the next version is taken through the table the roll-forward wrote
                _edit_in_the_record_tick(orc, layer, LT, rng, f"{tag} after the roll forward to {k}")

        # ---- retire the oldest increments: the next increment costs what it cost before
        if k == RETIRE_AT:
            nxt = SimpleNamespace(base=A(k), bt=TA(k), layer=layer, lt=LT)
            want_next = TS.expected_read(vm, orc, nxt, bb)
            for S, T in ((A, TA), (B, TB)):
                r = vm.retire_versions([(S(i), T(i)) for i in RETIRED], [(S(i), T(i)) for i in KEPT_AT_RETIRE],
                                       flags=f_store, **kw)
                # (records_stale is 0 where an unlink does not move the inode's ctime, as in some sandboxed kernels)
                assert r["versions_retired"] == len(RETIRED) and r["records_stale"] == r["records_restamped"], (ctx, r)
                for i in RETIRED:
                    assert not S(i).exists() and not T(i).exists(), ctx
                    state.pop(S(i))
            kept[:] = [v for v in kept if v not in RETIRED]
            assert TS.expected_read(vm, orc, nxt, bb) == want_next, ctx
            stores_unchanged(ctx + " after the retire")

    # ---- the stores as a whole
    pairs = {S: [(S(v), T(v)) for v in kept] for S, T in ((A, TA), (B, TB))}
    res = {S: vm.scrub_store(p, flags=f_store, **kw) for S, p in pairs.items()}
    for r in res.values():
        assert r["verdicts"] == [vm.VMIG_OK] * len(kept) and r["findings"] == [], (tag, r["verdicts"], r["findings"][:5])
    inodes = {}
    for v in kept:
        for key, (size, rel) in _regular_inodes(A(v)).items():
            inodes.setdefault(key, (size, set(), v, rel))[1].add(v)
    assert res[A]["bytes_unique"] == res[B]["bytes_unique"] == sum(x[0] for x in inodes.values()), tag

    # ---- one wrong byte in an A inode two kept versions share
    lpath = lambda rel: os.path.join(os.fsencode(os.fspath(layer)), rel)
    shared = sorted((kv for kv in inodes.items() if kv[1][0] > 0 and len(kv[1][1]) >= 2),
                    key=lambda kv: (len(kv[1][1]) == len(kept), kv[1][3]))
    pick = None
    for key, (size, versions, k0, rel) in shared:     # a version whose path of the inode the layer has as a regular file
        for v in sorted(versions, reverse=True):
            rel_v = _first_path(A(v), key)            # the path a rollback fetches; the group's others are linked to it
            if os.path.isfile(lpath(rel_v)) and not os.path.islink(lpath(rel_v)):
                pick = (size, versions, k0, rel, key, v, rel_v)
                break
        if pick:
            break
    assert pick, tag
    size, versions, k0, rel, key, j, rel_j = pick
    off = size // 2
    _flip_at(os.path.join(os.fsencode(os.fspath(A(k0))), rel), off, ROT)
    ctx = f"{tag}: damaged {rel!r} at {off}, linked by versions {sorted(versions)}"
    r = vm.scrub_store(pairs[A], flags=f_store, **kw)
    assert r["verdicts"] == [vm.VMIG_ECORRUPT if v in versions else vm.VMIG_OK for v in kept], (ctx, r["verdicts"])
    lo = off // bb * bb
    bad = Path(os.fsdecode(os.path.join(os.fsencode(os.fspath(A(j))), rel_j))).read_bytes()[lo:lo + bb]
    good = bytearray(bad)
    good[off - lo] ^= ROT
    with open(lpath(rel_j), "rb") as f:               # the layer must lack the good block, so that the rollback fetches it
        f.seek(lo)
        holds_good = f.read(len(good)) == bytes(good)
    if holds_good:
        _flip_at(lpath(rel_j), lo + (off - lo + 1) % len(good), 0xFF)
    table_before = LT.read_bytes()
    with pytest.raises(vm.VmigError) as ei:
        vm.rollback_layer(layer, A(j), TA(j), LT, LT, flags=F, **kw)
    assert ei.value.code == vm.VMIG_ECORRUPT, (ctx, ei.value)
    assert LT.read_bytes() == table_before, ctx
    for dp, _d, fns in os.walk(os.fsencode(os.fspath(layer))):
        for n in fns:
            p = os.path.join(dp, n)
            if stat.S_ISREG(os.lstat(p).st_mode):
                assert bad not in Path(os.fsdecode(p)).read_bytes(), (ctx, p)
    # a snapshot on the damaged version takes nothing from the damaged inode
    D, DT = root / "Adamaged", root / "Adamaged.vmig"
    D.mkdir()
    want = orc.block_table_of_tree(layer, bb)
    r = vm.snapshot_layer(layer, D, A(j), TA(j), DT, LT, flags=F, **kw)
    assert r["files_base_untrusted"] >= 1, (ctx, r)
    assert key not in _regular_inodes(D), ctx
    _table_is(orc, DT, want, ctx)
    tar = root / "tar"
    tar.mkdir()
    orc.ref_copy(layer, tar)
    TS.same_tree(orc, tar, D)
    r = vm.scrub_store([(D, DT)], flags=f_store, **kw)
    assert r["verdicts"] == [vm.VMIG_OK], (ctx, r["findings"][:5])
    print(f"{tag}: detours at {sorted(detours)}, {extras} files read by the prune exception "
          f"(an unlink moves ctime: {unlink_moves_ctime})")


# ------------------------------------------------------------------------------------------------ the hand-off mirror
def test_handoff_mirror_over_one_replicaset(vm, orc, shm_tmp):
    """handoff.py over rs-1 ... rs-6: each version is the hand-off of the previous container, the tenant's edits, and
    SnapshotVersionFromLayer, whose out table is the layer table's own path.  At two versions the new container is first
    compared with and rolled back to an older version and rolled forward again (RollbackInPlace rewrites its blocks.vmig),
    so that its snapshot is taken through a table a rollback wrote.  RetireVersions keeps three; ScrubReplicaSet ends."""
    ho = importlib.import_module(vm.__name__ + ".handoff")
    bb, seed, n = vm.BLOCK_BYTES, 41, 6
    ops = L.script(seed, n - 1, bb)                          # ops[v - 2] turns rs-(v-1)'s content into rs-v's
    rng = np.random.default_rng(seed)
    detours = set(int(x) for x in rng.choice([3, 4, 6], size=2, replace=False))
    ups = {f"rs-{v}": shm_tmp / f"upper_{v}" for v in range(1, n + 1)}
    for p in ups.values():
        p.mkdir()
    L.build_layer(ups["rs-1"], orc, bb, make_rich_tree)
    vm.set_resolver(container_upperdir=lambda name: str(ups[name]))
    ho.set_merges_root(shm_tmp)
    noop = lambda name: None

    def snapshot_matches_layer(name, ctx):
        data, table = ho.snapshotPaths(name)
        tar = shm_tmp / f"tar_{name}"
        tar.mkdir()
        orc.ref_copy(ups[name], tar)
        TS.same_tree(orc, tar, data)
        _table_is(orc, table, orc.block_table_of_tree(ups[name], bb), ctx)
        shutil.rmtree(tar)

    try:
        ho.SnapshotVersionFromLayer("rs-1")
        snapshot_matches_layer("rs-1", "rs-1")
        for v in range(2, n + 1):
            name, prev = f"rs-{v}", f"rs-{v - 1}"
            ctx = f"{name}: {json.dumps(ops[v - 2])}"
            ho.HandoffCopy(prev, name, pause=noop, resume=noop)
            _, table = ho.snapshotPaths(name)
            _table_is(orc, table, orc.block_table_of_tree(ups[name], bb), ctx + " hand-off")
            if v in detours:
                versions = ho.snapshotVersions("rs")
                target = versions[int(rng.integers(len(versions) - 1))]          # older than the one just handed off
                tdata, ttable = ho.snapshotPaths(target)
                want, c = TC.expected(ups[name], tdata, bb, 0, table)
                r = ho.CompareWithVersion(target, name, shm_tmp / "cmp.txt")
                assert (shm_tmp / "cmp.txt").read_bytes() == want and {x: r[x] for x in TC.COUNTERS} == c, (ctx, target)
                for to in (target, prev):                  # back, then forward to the content the hand-off brought
                    want_fetch, _second = TR.restore_bytes(ups[name], ho.snapshotPaths(to)[0], bb)
                    r = ho.RollbackInPlace(to, name)
                    assert r["bytes_fetched"] == want_fetch, (ctx, to, r)
                    assert L.diff_manifests(L.tree_in_itself(orc, ups[name]), L.tree_in_itself(orc, ho.snapshotPaths(to)[0])) == [], (ctx, to)
                    _table_is(orc, table, orc.block_table_of_tree(ups[name], bb), (ctx, to))
                    _identities_are_lstat(orc, table, ups[name], (ctx, to))
            L.apply(ups[name], ops[v - 2])
            r = ho.SnapshotVersionFromLayer(name)
            assert "files_trusted" in r, (ctx, r)                       # taken through the layer's table
            snapshot_matches_layer(name, ctx)
            if v == 5:
                before = ho.snapshotVersions("rs")
                r = ho.RetireVersions("rs", keep=3)
                assert r["retired"] == before[:-3] and r["kept"] == before[-3:] == ["rs-3", "rs-4", "rs-5"], r
                assert r["records_stale"] == r["records_restamped"], r
                assert ho.baseVersion("rs-6") == "rs-5" and not any(ho.versionDir(x).exists() for x in r["retired"])
        r = ho.ScrubReplicaSet("rs")
        assert r["verdicts"] == {f"rs-{v}": vm.VMIG_OK for v in range(3, n + 1)}, r
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
