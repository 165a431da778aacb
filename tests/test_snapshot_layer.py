"""vmig_snapshot_layer on the GPU (-m gpu).  Every call is held to vmig_snapshot_tree with the same arguments on an identical
layer and base built beside it (a snapshot's links move its base inodes' ctimes, so one base serves one call): the same
tree, the same path -> base-inode links, the same backfilled bytes, the same out table, and the same five counters, and
both to the tar copy of the layer.  The bytes read from the layer are restated here from the two tables and lstat."""
import importlib
import os
import shutil
import stat
import struct
import threading
import time
from pathlib import Path

import pytest

import _layer_model as lm
from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
SHARED = ("files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled", "files_base_untrusted")
T = 1_600_000_000_000_000_000            # the fixed mtime of every entry the second round of changes touches


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


def _populate(root: Path, orc, bb: int, rich: bool):
    (root / "m").mkdir()
    (root / "u").mkdir()
    sizes = {"m/a.bin": 5 * bb + 123, "m/b.bin": 3 * bb, "m/c.bin": 4 * bb + 7, "m/d.bin": 2 * bb + 11, "m/e.bin": 3 * bb + 1,
             "m/p.bin": 2 * bb + 3, "m/q.bin": 2 * bb + 3, "u/chmod.bin": 2 * bb, "u/edit2.bin": 3 * bb, "u/rewrite.bin": 2 * bb + 5,
             "u/append2.bin": bb + 9, "u/base_rot.bin": 2 * bb}
    sizes.update({f"u/keep{i}.bin": (i + 1) * bb + 17 * i for i in range(4)})
    for i, (rel, n) in enumerate(sorted(sizes.items())):
        (root / rel).write_bytes(lm.data(40 + i, n))
    (root / "u" / "dup.bin").write_bytes((root / "u" / "keep0.bin").read_bytes())
    if rich:
        (root / "rich").mkdir()
        make_rich_tree(root / "rich", orc, big=2 * bb + 777)


def _phase1(root: Path, bb: int):
    """Changes made before the layer's table was written: the table vouches for their result."""
    _flip(root / "m" / "a.bin", 2 * bb + 5)                                    # in-place block edit
    with open(root / "m" / "b.bin", "ab") as f:                                # append
        f.write(lm.data(90, bb // 2 + 3))
    os.truncate(root / "m" / "c.bin", 2 * bb + 5)                              # truncate
    os.unlink(root / "m" / "d.bin")                                            # deletion
    (root / "n").mkdir()
    os.rename(root / "m" / "e.bin", root / "n" / "e_moved.bin")                # rename, mtime kept
    os.rename(root / "m" / "p.bin", root / "m" / "tmp")                        # swapped pair
    os.rename(root / "m" / "q.bin", root / "m" / "p.bin")
    os.rename(root / "m" / "tmp", root / "m" / "q.bin")
    (root / "n" / "new1.bin").write_bytes(lm.data(91, 2 * bb + 9))             # new file


def _phase2(root: Path, bb: int):
    """Changes made after the layer's table was written: the table no longer vouches for these files."""
    os.chmod(root / "u" / "chmod.bin", 0o600)                                  # chmod only
    _flip(root / "u" / "edit2.bin", bb + 1)
    p = root / "u" / "rewrite.bin"                                             # the same size, rewritten
    p.write_bytes(lm.data(92, p.stat().st_size))
    with open(root / "u" / "append2.bin", "ab") as f:
        f.write(b"tail")
    (root / "n" / "new2.bin").write_bytes(lm.data(93, bb + 1))
    (root / "n" / "hl_a").write_bytes(lm.data(94, bb + 2))                     # hard-link pair
    os.link(root / "n" / "hl_a", root / "n" / "hl_b")
    os.symlink("../m/a.bin", root / "n" / "sym")
    os.mkfifo(root / "n" / "fifo")
    (root / "n" / "empty").write_bytes(b"")
    for rel in ("u/chmod.bin", "u/edit2.bin", "u/rewrite.bin", "u/append2.bin", "n/new2.bin", "n/hl_a", "n/empty"):
        os.utime(root / rel, ns=(T, T))
    os.utime(root / "n" / "sym", ns=(T, T), follow_symlinks=False)
    os.utime(root / "n" / "fifo", ns=(T, T))
    for dp, _, _ in os.walk(root):
        os.utime(dp, ns=(T, T))


class Setup:
    def __init__(self, root: Path, k: int):
        self.base, self.bt = root / f"base{k}", root / f"base{k}.vmig"
        self.layer, self.lt = root / f"layer{k}", root / f"layer{k}.vmig"
        self.dst, self.out = root / f"dst{k}", root / f"dst{k}.vmig"


def build(vm, orc, root: Path, bb: int, n: int, rich: bool = True, phase2: bool = True, changes: bool = True):
    """n identical (base snapshot, layer, layer table) sets: the base is a snapshot of the first state, the layer a
    migration of the state after the first round of changes (its table written by that migration), then changed again."""
    s0, s1 = root / "s0", root / "s1"
    s0.mkdir()
    _populate(s0, orc, bb, rich)
    lm.freeze(s0, s1)
    if changes:
        _phase1(s1, bb)
    sets = []
    for k in range(n):
        s = Setup(root, k)
        s.base.mkdir()
        vm.snapshot_tree(s0, s.base, None, None, s.bt, block_bytes=bb)
        s.layer.mkdir()
        vm.migrate_tree(s1, s.layer, None, s.lt, block_bytes=bb)
        if changes and phase2:
            _phase2(s.layer, bb)
        s.dst.mkdir()
        sets.append(s)
    return sets


def _regular_primaries(root: Path):
    """rel (bytes) -> lstat of each regular file that is the first path (bytewise) of its in-tree inode group."""
    root = os.fsencode(os.fspath(root))
    seen, out = set(), {}
    paths = []
    for dp, _, fns in os.walk(root):
        for n in fns:
            paths.append(os.path.relpath(os.path.join(dp, n), root))
    for rel in sorted(paths):
        st = os.lstat(os.path.join(root, rel))
        if stat.S_ISREG(st.st_mode) and st.st_ino not in seen:
            seen.add(st.st_ino)
            out[rel] = st
    return out


def expected_read(vm, orc, s: Setup, bb: int, layer_table=None) -> tuple:
    """(files trusted, bytes read) by include/vmig.h: a trusted layer file reads the blocks of its record whose (hash,
    length) no trusted base file holds; every other regular file is read in full."""
    lt = layer_table or s.lt
    B, bh = orc.read_table(s.bt), vm.table_hashes(s.bt)
    index = set()
    for (rel, size, first), (ino, ct) in zip(B["entries"], B["identity"]):
        try:
            st = os.lstat(os.path.join(os.fsencode(os.fspath(s.base)), rel))
        except FileNotFoundError:
            continue
        if ino and stat.S_ISREG(st.st_mode) and (st.st_ino, st.st_size, st.st_ctime_ns) == (ino, size, ct):
            index |= {(int(bh[first + r]), min(bb, size - r * bb)) for r in range(-(-size // bb))}
    L, lh = orc.read_table(lt), vm.table_hashes(lt)
    rec = {rel: (size, first, ino, ct) for (rel, size, first), (ino, ct) in zip(L["entries"], L["identity"])}
    trusted = read = 0
    for rel, st in _regular_primaries(s.layer).items():
        if not st.st_size:
            continue
        r = rec.get(rel)
        if r and r[2] and (st.st_ino, st.st_size, st.st_ctime_ns) == (r[2], r[0], r[3]):
            trusted += 1
            read += sum(min(bb, st.st_size - i * bb) for i in range(-(-st.st_size // bb))
                        if (int(lh[r[1] + i]), min(bb, st.st_size - i * bb)) not in index)
        else:
            read += st.st_size
    return trusted, read


def links(dst: Path, base: Path) -> dict:
    """rel -> the base path whose inode the snapshot's path is (None: a new inode)."""
    by_ino = {st.st_ino: rel for rel, st in _regular_primaries(base).items()}
    return {rel: by_ino.get(st.st_ino) for rel, st in _regular_primaries(dst).items()}


def layer_state(root: Path, bodies: bool = True) -> dict:
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in [""] + dns + fns:
            p = os.path.join(dp, n) if n else dp
            st = os.lstat(p)
            body = Path(p).read_bytes() if bodies and stat.S_ISREG(st.st_mode) else st.st_size
            out[p] = (st.st_ino, st.st_mode, st.st_mtime_ns, st.st_ctime_ns, body)
    return out


def same_tree(orc, a, b):
    assert lm.diff_manifests(lm.tree_in_itself(orc, a), lm.tree_in_itself(orc, b)) == []


def check_pair(vm, orc, ref: Setup, new: Setup, r_tree: dict, r_layer: dict, bb: int, flags: int, restore=True):
    """The layer call's snapshot against the tree call's on an identical setup, and both against the tar copy."""
    same_tree(orc, ref.dst, new.dst)
    tar = new.dst.with_name("tar_" + new.dst.name)
    tar.mkdir()
    orc.ref_copy(new.layer, tar)
    same_tree(orc, tar, new.dst)
    assert links(ref.dst, ref.base) == links(new.dst, new.base)
    a, b = orc.read_table(ref.out), orc.read_table(new.out)
    assert a["entries"] == b["entries"] and (vm.table_hashes(ref.out) == vm.table_hashes(new.out)).all()
    _, want = orc.block_table_of_tree(new.layer, bb)
    assert (vm.table_hashes(new.out) == want).all()
    assert {k: r_tree[k] for k in SHARED} == {k: r_layer[k] for k in SHARED}, (r_tree, r_layer)
    if restore:
        back = new.dst.with_name("restore_" + new.dst.name)
        back.mkdir()
        vm.restore_tree(new.dst, new.out, back, None, None, flags=vm.F_VERIFY, block_bytes=bb)
        assert orc.compare_trees(tar, back) == []
        shutil.rmtree(back)
    shutil.rmtree(tar)


def written_bytes(s: Setup) -> int:
    """Sizes of the snapshot's inodes that are not base inodes: what F_VERIFY re-reads."""
    base = {st.st_ino for st in _regular_primaries(s.base).values()}
    return sum(st.st_size for st in _regular_primaries(s.dst).values() if st.st_ino not in base)


def run_pair(vm, orc, ref: Setup, new: Setup, bb: int, flags: int, lanes: int = 1, layer_table=None, restore=True):
    trusted, want_read = expected_read(vm, orc, new, bb, layer_table)
    before = layer_state(new.layer)
    r_tree = vm.snapshot_tree(ref.layer, ref.dst, ref.base, ref.bt, ref.out, flags=flags, block_bytes=bb, lanes_per_gpu=lanes)
    r = vm.snapshot_layer(new.layer, new.dst, new.base, new.bt, new.out, layer_table or new.lt, flags=flags, block_bytes=bb,
                          lanes_per_gpu=lanes)
    assert layer_state(new.layer) == before
    assert r["files_trusted"] == trusted and r["bytes_read"] == want_read, (r, trusted, want_read)
    if flags & vm.F_VERIFY:
        assert r["bytes_h2d"] == r["bytes_read"] + written_bytes(new), r
    else:
        assert r["bytes_h2d"] == r["bytes_read"], r
    assert r["bytes_total"] == r["bytes_read"]
    check_pair(vm, orc, ref, new, r_tree, r, bb, flags, restore)
    return r_tree, r


# ------------------------------------------------------------------------------------------ 1. equivalence
@pytest.mark.parametrize("bb,lanes,flags,disk", [(4 << 20, 1, "verify", False), (65536, 3, "none", False),
                                                 ((1 << 20) + 4096, 3, "verify", False), (4 << 20, 3, "direct", True)])
def test_layer_snapshot_equals_tree_snapshot(vm, orc, shm_tmp, tmp_path, bb, lanes, flags, disk):
    root = tmp_path if disk else shm_tmp
    f = {"verify": vm.F_VERIFY, "none": 0, "direct": vm.F_VERIFY | vm.F_DIRECT_IO}[flags]
    ref, new = build(vm, orc, root, bb, 2)
    _, r = run_pair(vm, orc, ref, new, bb, f, lanes)
    layer_bytes = sum(st.st_size for st in _regular_primaries(new.layer).values())
    assert r["files_trusted"] > 0 and 0 < r["bytes_read"] < layer_bytes // 2
    assert r["files_linked"] > 0 and r["files_backfilled"] > 0
    # the renamed file and the unchanged ones are links to the base; the swapped pair too
    ln = links(new.dst, new.base)
    assert ln[b"n/e_moved.bin"] == b"m/e.bin" and ln[b"u/keep1.bin"] == b"u/keep1.bin"
    assert ln[b"m/p.bin"] == b"m/q.bin" and ln[b"m/q.bin"] == b"m/p.bin"
    assert ln[b"u/rewrite.bin"] is None and ln[b"u/chmod.bin"] is None


# ------------------------------------------------------------------------------------------ 2. cost
def test_unchanged_layer_reads_nothing_and_links_every_solo_file(vm, orc, shm_tmp):
    bb = 1 << 20
    ref, new = build(vm, orc, shm_tmp, bb, 2, rich=False, changes=False)
    r_tree, r = run_pair(vm, orc, ref, new, bb, 0)
    solo = [rel for rel, st in _regular_primaries(new.layer).items() if st.st_size and st.st_nlink == 1]
    assert r["bytes_h2d"] == 0 and r["bytes_read"] == 0 and r["files_read"] == 0
    assert r["files_linked"] == len(solo) == r["files_trusted"] and r_tree["bytes_h2d"] > 0
    assert all(links(new.dst, new.base)[rel] is not None for rel in solo)


# ------------------------------------------------------------------------------------------ 3. trust edges
def _format01(src: Path, dst: Path):
    """The same table in format 01: no identities."""
    raw = src.read_bytes()
    bb, algo, nf, nb = struct.unpack_from("<IIQQ", raw, 8)
    out, off = bytearray(b"VMIGBT01" + raw[8:32]), 32
    for _ in range(nf):
        (pl,) = struct.unpack_from("<I", raw, off)
        out += raw[off:off + 4 + pl + 16]
        off += 4 + pl + 32
    out += raw[off:]
    dst.write_bytes(bytes(out))


def test_tables_that_trust_nothing_and_a_rewritten_base_file(vm, orc, shm_tmp):
    bb = 1 << 20
    sets = build(vm, orc, shm_tmp, bb, 6, rich=False)
    # a format-01 layer table, and the base's own table passed as the layer's: nothing trusted, the same result
    _format01(sets[1].lt, shm_tmp / "v1.vmig")
    for ref, new, lt in ((sets[0], sets[1], shm_tmp / "v1.vmig"), (sets[2], sets[3], sets[3].bt)):
        _, r = run_pair(vm, orc, ref, new, bb, vm.F_VERIFY, layer_table=lt, restore=False)
        assert r["files_trusted"] == 0 and r["bytes_read"] == sum(st.st_size for st in _regular_primaries(new.layer).values())
    # a base file rewritten (same size) before the call: its blocks are read from the layer
    ref, new = sets[4], sets[5]
    for s in (ref, new):
        p = s.base / "u" / "base_rot.bin"
        p.write_bytes(lm.data(777, p.stat().st_size))
    _, r = run_pair(vm, orc, ref, new, bb, vm.F_VERIFY)
    assert r["files_base_untrusted"] >= 1 and links(new.dst, new.base)[b"u/base_rot.bin"] is None


def test_stale_record_fails_with_esrcchanged(vm, orc, shm_tmp):
    bb = 1 << 20
    (s,) = build(vm, orc, shm_tmp, bb, 1, rich=False)
    t = orc.read_table(s.lt)
    first = next(f for rel, _, f in t["entries"] if rel == b"u/keep1.bin")
    raw = bytearray(s.lt.read_bytes())
    off = len(raw) - 8 * (len(t["hashes"]) - first)
    raw[off] ^= 1                                                  # a hash no base block has: the block must be read
    s.lt.write_bytes(bytes(raw))
    before, table = layer_state(s.layer), bytes(raw)
    with pytest.raises(vm.VmigError) as ei:
        vm.snapshot_layer(s.layer, s.dst, s.base, s.bt, s.out, s.lt, flags=vm.F_VERIFY, block_bytes=bb)
    assert ei.value.code == vm.VMIG_ESRCCHANGED and "u/keep1.bin block 0" in str(ei.value), ei.value
    assert not any(n.startswith(s.out.name) for n in os.listdir(s.out.parent))
    assert layer_state(s.layer) == before and s.lt.read_bytes() == table


# ------------------------------------------------------------------------------------------ 4. cancel, concurrency
def test_cancel_then_succeed(vm, orc, shm_tmp):
    bb = 4 << 20
    src, base, layer = shm_tmp / "src", shm_tmp / "base", shm_tmp / "layer"
    src.mkdir()
    for i in range(12):
        (src / f"f{i:02d}").write_bytes(lm.data(3 + i, 96 * MiB))
    base.mkdir()
    vm.snapshot_tree(src, base, None, None, shm_tmp / "base.vmig", block_bytes=bb)
    lm.freeze(src, layer)
    for i in range(12):
        _flip(layer / f"f{i:02d}", (i % 20) * bb + 3)
    before = layer_state(layer, bodies=False)
    # the base's own table as the layer's trusts nothing: every byte of the layer is read
    args = lambda d: (layer, d, base, shm_tmp / "base.vmig", shm_tmp / "out.vmig", shm_tmp / "base.vmig")
    (shm_tmp / "d0").mkdir()
    with vm.Ctl() as c:
        c.cancel()
        with pytest.raises(vm.VmigError) as ei:
            vm.snapshot_layer(*args(shm_tmp / "d0"), block_bytes=bb, ctl=c)
        assert ei.value.code == vm.VMIG_ECANCELED and os.listdir(shm_tmp / "d0") == []
    hit = False
    for k in range(1, 4):
        d = shm_tmp / f"d{k}"
        d.mkdir()
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
                vm.snapshot_layer(*args(d), flags=vm.F_VERIFY, block_bytes=bb, ctl=c)
                os.unlink(shm_tmp / "out.vmig")                        # the pass was too short to hit: start over
            except vm.VmigError as e:
                assert e.code == vm.VMIG_ECANCELED and "cancelled in phase DATA" in str(e), e
                hit = True
            finally:
                done.set()
                th.join()
        assert not any(n.startswith("out.vmig") for n in os.listdir(shm_tmp))
        assert layer_state(layer, bodies=False) == before
        if hit:
            break
    assert hit, "a cancel half way through the data pass was not honoured"
    d = shm_tmp / "dok"
    d.mkdir()
    vm.snapshot_layer(*args(d), flags=vm.F_VERIFY, block_bytes=bb)
    same_tree(orc, layer, d)


def test_two_layer_snapshots_and_a_tree_snapshot_at_once(vm, orc, shm_tmp):
    bb = 1 << 20
    groups = []
    for g in range(3):
        root = shm_tmp / f"g{g}"
        root.mkdir()
        groups.append(build(vm, orc, root, bb, 2, rich=(g == 0)))
    errs, out = [], {}

    def run(name, fn):
        try:
            out[name] = fn()
        except Exception as e:                       # noqa: BLE001 -- reported below
            errs.append((name, e))
    calls = {
        0: lambda s: vm.snapshot_layer(s.layer, s.dst, s.base, s.bt, s.out, s.lt, flags=vm.F_VERIFY, block_bytes=bb, lanes_per_gpu=2),
        1: lambda s: vm.snapshot_layer(s.layer, s.dst, s.base, s.bt, s.out, s.lt, block_bytes=bb),
        2: lambda s: vm.snapshot_tree(s.layer, s.dst, s.base, s.bt, s.out, flags=vm.F_VERIFY, block_bytes=bb),
    }
    ths = [threading.Thread(target=run, args=(g, lambda g=g: calls[g](groups[g][0]))) for g in range(3)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errs, errs
    for g in range(3):
        conc, serial = groups[g]
        r = calls[g](serial)
        same_tree(orc, conc.dst, serial.dst)
        assert links(conc.dst, conc.base) == links(serial.dst, serial.base)
        assert (vm.table_hashes(conc.out) == vm.table_hashes(serial.out)).all()
        assert {k: out[g][k] for k in SHARED} == {k: r[k] for k in SHARED}


# ------------------------------------------------------------------------------------------ 5. the hand-off mirror
def test_handoff_chain_from_layer(vm, orc, shm_tmp):
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {f"rs-{i}": shm_tmp / f"upper_{i}" for i in (1, 2, 3)}
    for p in ups.values():
        p.mkdir()
    for i in range(4):
        (ups["rs-1"] / f"g{i}.bin").write_bytes(lm.data(300 + i, 9 * MiB + i))
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        r1 = ho.SnapshotVersionFromLayer("rs-1")                   # no base, no table: SnapshotVersionIncremental
        assert r1.get("files_linked", 0) == 0 and "files_trusted" not in r1
        for v, edit in ((2, "g1.bin"), (3, "g2.bin")):
            prev, cur = f"rs-{v - 1}", f"rs-{v}"
            _, table = ho.snapshotPaths(cur)
            table.parent.mkdir(parents=True)
            ho.CopyDirDiffVerified(ups[prev], ups[cur], None, table)     # the hand-off's table for the new layer
            _flip(ups[cur] / edit, 5 * MiB)
            r = ho.SnapshotVersionFromLayer(cur)
            assert r["files_trusted"] == 3 and r["bytes_read"] == 9 * MiB + int(edit[1]), r
            data, table = ho.snapshotPaths(cur)
            ref = shm_tmp / f"ref_{v}"
            ref.mkdir()
            orc.ref_copy(ups[cur], ref)
            same_tree(orc, ref, data)
            _, want = orc.block_table_of_tree(ups[cur])
            assert (vm.table_hashes(table) == want).all()
            back = shm_tmp / f"back_{v}"
            back.mkdir()
            vm.restore_tree(data, table, back, None, None, flags=vm.F_VERIFY)
            assert orc.compare_trees(ref, back) == []
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
