"""One layer through many versions on the GPU (-m gpu), differential against the reference's tar pipe at every step.

The destination, the prior table and the snapshot store carry state from one call into the next, so each chain below
applies nine versions of one seeded layer (tests/_layer_model.py) to ONE destination: the plain call against tar's own
evolving destination, the hand-off call (prune + verify) against a fresh tar copy, incremental snapshots against frozen
copies of every version, then scrub and rollback across arbitrary distance.  The kind-change matrix runs every ordered
pair of entry kinds at one path singly and holds the engine to what GNU tar does (test_versions_host.py pins that)."""
import json
import os
import shutil
import stat
from pathlib import Path

import numpy as np
import pytest

import _layer_model as L
from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
N = 8


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _fresh(p: Path) -> Path:
    shutil.rmtree(p, ignore_errors=True)
    p.mkdir()
    return p


def _frozen(orc, root: Path, mtime_ns: bool = False) -> dict:
    """The manifest a copy of the frozen version `root` must have.  As root that is the version itself; an ordinary
    user's tar, and so the engine, applies the umask and keeps no set-id or sticky bit."""
    man = L.tree_in_itself(orc, root, mtime_ns)
    if os.geteuid() != 0:
        um = os.umask(0)
        os.umask(um)
        for r in man.values():
            if not stat.S_ISLNK(r["type"]):
                r["mode"] &= 0o777 & ~um
    return man


def _check_table(orc, table: Path, want, dst: Path, second: set, snapshot: bool, ctx):
    """The table the call wrote is the oracle's, and the identities in it are those of the files the call left."""
    got = orc.read_table(table)
    entries, hashes = want
    assert got["entries"] == entries, ctx
    wrong = np.flatnonzero(got["hashes"] != hashes)
    assert wrong.size == 0, (ctx, [rel for rel, size, first in entries if size and first <= wrong[0]][-1:])
    for (rel, _size, _first), (ino, ctime_ns) in zip(entries, got["identity"]):
        st = os.lstat(os.path.join(os.fsencode(dst), rel))
        if rel in second:                          # a later path of a hard-link group is never patched in place
            assert (ino, ctime_ns) == (0, 0), (ctx, rel)
        else:
            assert ino == st.st_ino, (ctx, rel)
            # (a group's first path got its links after a plain call recorded it; a snapshot records it afterwards)
            if st.st_nlink == 1 or snapshot:
                assert ctime_ns == st.st_ctime_ns, (ctx, rel)


def _regular_inodes(root: Path) -> dict:
    out = {}
    for dirpath, _d, files in os.walk(os.fsencode(root)):
        for n in files:
            st = os.lstat(os.path.join(dirpath, n))
            if stat.S_ISREG(st.st_mode):
                out.setdefault((st.st_dev, st.st_ino), (st.st_size, os.path.relpath(os.path.join(dirpath, n), os.fsencode(root))))
    return out


# ------------------------------------------------------------------------------------------------ the sequence
@pytest.mark.parametrize("seed,bb,lanes", [(11, 65536, 1), (12, 65536, 1), (13, 65536, 1), (14, 65536, 3),
                                           (15, 4 << 20, 1), (16, 4096, 1)])
def test_one_layer_through_nine_versions(vm, orc, shm_tmp, seed, bb, lanes):
    kw = dict(block_bytes=bb, lanes_per_gpu=lanes)
    src = shm_tmp / "src"
    L.build_layer(src, orc, bb, make_rich_tree)
    ops = [[]] + L.script(seed, N, bb)                       # version 0 is the layer as built
    dstA, refA, dstB = _fresh(shm_tmp / "dstA"), _fresh(shm_tmp / "refA"), _fresh(shm_tmp / "dstB")
    T = lambda name, k: shm_tmp / f"{name}{k}.vmig"
    S = [shm_tmp / f"S{k}" for k in range(N + 1)]
    frozen = [shm_tmp / f"frozen{k}" for k in range(N + 1)]
    man, otab, snap_state = [], [], []
    for k in range(N + 1):
        ctx = f"seed {seed} bb {bb} lanes {lanes} version {k}: {json.dumps(ops[k])}"
        L.apply(src, ops[k])
        L.freeze(src, frozen[k])
        man.append(L.tree_in_itself(orc, src))
        otab.append(orc.block_table_of_tree(src, bb))
        second = L.secondaries(man[k])
        second_blocks = sum(-(-size // bb) for rel, size, _ in otab[k][0] if rel in second)
        trusted = L.single_files(man[k - 1]) if k else set()
        want = L.expected_written(otab[k - 1] if k else None, otab[k], second, trusted, bb)
        fresh = _fresh(shm_tmp / "fresh")
        orc.ref_copy(src, fresh)
        want_fresh = L.tree_in_itself(orc, fresh)

        # ---- the plain call, against tar's own evolving destination: extras stay exactly where tar leaves them
        st = vm.migrate_tree(src, dstA, T("A", k - 1) if k else None, T("A", k), **kw)
        orc.ref_copy(src, refA)
        assert orc.compare_trees(refA, dstA) == [], ctx
        _check_table(orc, T("A", k), otab[k], dstA, second, False, ctx)
        assert (st["blocks_total"] - st["blocks_skipped"] - second_blocks, st["bytes_written"]) == want, (ctx, st)

        # ---- the hand-off's final pass, against a fresh tar copy
        st = vm.migrate_tree(src, dstB, T("B", k - 1) if k else None, T("B", k), flags=vm.F_PRUNE | vm.F_VERIFY, **kw)
        assert L.diff_manifests(want_fresh, L.tree_in_itself(orc, dstB)) == [], ctx
        _check_table(orc, T("B", k), otab[k], dstB, second, False, ctx)
        assert (st["blocks_total"] - st["blocks_skipped"] - second_blocks, st["bytes_written"]) == want, (ctx, st)
        assert st["pruned"] == (L.expected_pruned(man[k - 1], man[k]) if k else 0), (ctx, st)

        # ---- an incremental snapshot on the previous one
        S[k].mkdir()
        st = vm.snapshot_tree(src, S[k], S[k - 1] if k else None, T("S", k - 1) if k else None, T("S", k),
                              flags=vm.F_VERIFY, **kw)
        snap_state.append(L.tree_in_itself(orc, S[k], mtime_ns=True))
        assert L.diff_manifests(want_fresh, L.tree_in_itself(orc, S[k])) == [], ctx
        _check_table(orc, T("S", k), otab[k], S[k], second, True, ctx)
        # nothing comes through the ring that any base block could supply
        assert st["bytes_written"] == L.expected_ring_bytes(otab[k - 1] if k else None, otab[k], second, bb), (ctx, st)
        base_inodes = _regular_inodes(S[k - 1]) if k else {}
        shared = [v for key, v in _regular_inodes(S[k]).items() if key in base_inodes]
        assert (st["files_linked"], st["bytes_linked"]) == (len(shared), sum(s for s, _ in shared)), (ctx, st)
        assert st["files_base_untrusted"] == 0, (ctx, st)
        # an increment never edits history: every earlier snapshot is what it was when it was taken
        for i in range(k):
            assert L.diff_manifests(snap_state[i], L.tree_in_itself(orc, S[i], mtime_ns=True)) == [], (ctx, f"snapshot {i}")
        assert L.diff_manifests(_frozen(orc, frozen[k]), L.tree_in_itself(orc, S[k])) == [], ctx

    # ---- the store as a whole
    tag = f"seed {seed} bb {bb} lanes {lanes}"
    pairs = [(S[k], T("S", k)) for k in range(N + 1)]
    r = vm.scrub_store(pairs, **kw)
    assert r["verdicts"] == [vm.VMIG_OK] * (N + 1) and r["findings"] == [], (tag, r["verdicts"], r["findings"][:5])
    inodes = {}
    for k in range(N + 1):
        for key, (size, rel) in _regular_inodes(S[k]).items():
            inodes.setdefault(key, (size, set(), k, rel))[1].add(k)
    assert r["bytes_unique"] == sum(v[0] for v in inodes.values()), tag

    # ---- rollback across arbitrary distance over ONE live directory, kinds changing in both directions
    live = _fresh(shm_tmp / "live")
    order = [int(j) for j in np.random.default_rng(seed).permutation(N + 1)]
    cur = None
    for step, j in enumerate(order):
        ctx = f"{tag} rollback {order[:step + 1]} (version {cur} -> {j}); version {j}: {json.dumps(ops[j])}"
        st = vm.restore_tree(S[j], T("S", j), live, T("L", step - 1) if step else None, T("L", step),
                             flags=vm.F_PRUNE | vm.F_VERIFY, **kw)
        assert L.diff_manifests(_frozen(orc, frozen[j]), L.tree_in_itself(orc, live)) == [], ctx
        second = L.secondaries(man[j])
        second_blocks = sum(-(-size // bb) for rel, size, _ in otab[j][0] if rel in second)
        want = L.expected_written(otab[cur] if step else None, otab[j], second, L.single_files(man[cur]) if step else set(), bb)
        assert (st["blocks_total"] - st["blocks_skipped"] - second_blocks, st["bytes_written"]) == want, (ctx, st)
        assert st["pruned"] == (L.expected_pruned(man[cur], man[j]) if step else 0), (ctx, st)
        cur = j

    # ---- one wrong byte in one shared inode: exactly the versions that link it are damaged, and none of them restores
    shared = sorted((v for v in inodes.values() if v[0] > 0 and 2 <= len(v[1])), key=lambda v: (len(v[1]) == N + 1, v[3]))
    assert shared, tag
    size, versions, k0, rel = shared[0]
    with open(os.path.join(os.fsencode(S[k0]), rel), "r+b") as f:
        f.seek(size // 2)
        c = f.read(1)
        f.seek(size // 2)
        f.write(bytes([c[0] ^ 1]))
    r = vm.scrub_store(pairs, **kw)
    ctx = f"{tag}: damaged {rel!r}, linked by versions {sorted(versions)}"
    assert r["verdicts"] == [vm.VMIG_ECORRUPT if k in versions else vm.VMIG_OK for k in range(N + 1)], (ctx, r["verdicts"])
    j = cur if cur in versions else min(versions)
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(S[j], T("S", j), live, T("L", N), T("L", "bad"), flags=vm.F_PRUNE | vm.F_VERIFY, **kw)
    assert ei.value.code == vm.VMIG_ECORRUPT and not T("L", "bad").exists(), (ctx, ei.value)
    # the damaged block never reaches the live layer, under any path a version has for that inode
    st = os.lstat(os.path.join(os.fsencode(S[k0]), rel))
    lo = size // 2 // bb * bb
    bad = Path(os.fsdecode(os.path.join(os.fsencode(S[k0]), rel))).read_bytes()[lo:lo + bb]
    for v in versions:
        p = os.path.join(os.fsencode(live), _regular_inodes(S[v])[(st.st_dev, st.st_ino)][1])
        if os.path.isfile(p) and not os.path.islink(p):
            with open(p, "rb") as f:
                f.seek(lo)
                assert f.read(bb) != bad, (ctx, p)


# ------------------------------------------------------------------------------------------------ the kind matrix, singly
BBK = 65536
KP = L.KIND_PATH


def _old_state(vm, orc, old_src: Path, dst: Path, table=None):
    """The destination holds the old version: by tar, or by the engine where the call under test takes a prior table."""
    _fresh(dst)
    if table is None:
        orc.ref_copy(old_src, dst)
    else:
        vm.migrate_tree(old_src, dst, None, table, block_bytes=BBK)


def _expect_path_error(vm, call, ctx):
    with pytest.raises(vm.VmigError) as ei:
        call()
    assert KP in str(ei.value), (ctx, ei.value)


@pytest.mark.parametrize("old,new", [(a, b) for a in L.KINDS for b in L.KINDS], ids=lambda k: k)
def test_kind_change_at_one_path(vm, orc, shm_tmp, old, new):
    tar_ok = (old, new) not in L.TAR_REFUSES
    variant = (L.KINDS.index(old) + L.KINDS.index(new)) % 3
    old_src, src = shm_tmp / "old", shm_tmp / "src"
    L.kind_tree(old_src, old, 30 + variant)
    L.kind_tree(src, new, 61 + variant)
    want_table = orc.block_table_of_tree(src, BBK)
    second = L.secondaries(L.tree_in_itself(orc, src))
    fresh = _fresh(shm_tmp / "fresh")
    orc.ref_copy(src, fresh)
    tar = _fresh(shm_tmp / "tar")                            # what the reference leaves: the pipe over the old state
    orc.ref_copy(old_src, tar)
    assert (orc.ref_copy(src, tar, check=False).returncode == 0) == tar_ok
    want_tar, want_fresh = L.tree_in_itself(orc, tar), L.tree_in_itself(orc, fresh)
    dst, prior, out = shm_tmp / "dst", shm_tmp / "prior.vmig", shm_tmp / "out.vmig"

    def done(ctx, want):
        assert L.diff_manifests(want, L.tree_in_itself(orc, dst)) == [], ctx
        _check_table(orc, out, want_table, dst, second, ctx.startswith("snapshot"), ctx)
        out.unlink()

    # ---- migrate_tree: plain, with a prior table of the old state, and pruning
    for mode in ("plain", "prior", "prune"):
        ctx = f"migrate {mode}: {old} -> {new} at {KP}"
        _old_state(vm, orc, old_src, dst, None if mode == "plain" else prior)
        before = prior.read_bytes() if mode != "plain" else None
        call = lambda: vm.migrate_tree(src, dst, None if mode == "plain" else prior, out, block_bytes=BBK,
                                       flags=vm.F_PRUNE if mode == "prune" else 0)
        if mode == "prune" or tar_ok:
            call()
            done(ctx, want_fresh if mode == "prune" else want_tar)
        else:
            _expect_path_error(vm, call, ctx)
            assert not out.exists(), ctx
        assert before is None or prior.read_bytes() == before, ctx

    # ---- snapshot_tree into what an abandoned attempt left, on a base that already holds every file of the source
    base, tbase = _fresh(shm_tmp / "base"), shm_tmp / "base.vmig"
    vm.snapshot_tree(src, base, None, None, tbase, block_bytes=BBK)
    base_state = L.tree_in_itself(orc, base, mtime_ns=True)
    for flags in (0, vm.F_PRUNE):
        ctx = f"snapshot flags {flags:#x}: {old} -> {new} at {KP}"
        _old_state(vm, orc, old_src, dst)
        call = lambda: vm.snapshot_tree(src, dst, base, tbase, out, block_bytes=BBK, flags=flags | vm.F_VERIFY)
        if flags or tar_ok:
            st = call()
            assert st["bytes_written"] == 0, (ctx, st)        # the base has every block
            done(ctx, want_fresh if flags else want_tar)
        else:
            _expect_path_error(vm, call, ctx)
            assert not out.exists(), ctx
        assert L.diff_manifests(base_state, L.tree_in_itself(orc, base, mtime_ns=True)) == [], ctx

    # ---- restore_tree of that base over the old state
    for flags in (0, vm.F_PRUNE):
        ctx = f"restore flags {flags:#x}: {old} -> {new} at {KP}"
        _old_state(vm, orc, old_src, dst)
        call = lambda: vm.restore_tree(base, tbase, dst, None, out, block_bytes=BBK, flags=flags | vm.F_VERIFY)
        if flags or tar_ok:
            call()
            done(ctx, want_fresh if flags else want_tar)
        else:
            _expect_path_error(vm, call, ctx)
            assert not out.exists(), ctx
