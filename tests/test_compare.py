"""vmig_compare_snapshot on the GPU (-m gpu).  Its oracle is restated here from os.lstat, oracle.hash_file and in-tree
hard-link grouping: the expected report byte for byte, every counter, and the read plan (shared inode, trusted record of
the layer's table, or a read of each distinct inode)."""
import importlib
import os
import shutil
import stat
import threading
import time
from pathlib import Path

import pytest

import _layer_model as lm
from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
TYPE = {stat.S_IFREG: b"f", stat.S_IFDIR: b"d", stat.S_IFLNK: b"l", stat.S_IFCHR: b"c", stat.S_IFBLK: b"b", stat.S_IFIFO: b"p"}
COUNTERS = ("paths_added", "paths_removed", "paths_changed", "files_changed", "blocks_changed", "bytes_restore",
            "files_read", "bytes_read", "files_trusted", "files_shared")


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


# ------------------------------------------------------------------------------------------ the oracle
def _walk(root, skip_hidden=False) -> dict:
    """rel (bytes) -> lstat of every entry ("." is the root); sockets skipped, as the engine skips them."""
    root = os.fsencode(os.fspath(root))
    out = {b".": os.lstat(root)}

    def rec(d, rel, depth):
        for n in sorted(os.listdir(d)):
            p = os.path.join(d, n)
            st = os.lstat(p)
            if stat.S_ISSOCK(st.st_mode) or (stat.S_ISDIR(st.st_mode) and skip_hidden and depth == 0 and n.startswith(b".")):
                continue
            r = n if rel == b"." else rel + b"/" + n
            out[r] = st
            if stat.S_ISDIR(st.st_mode):
                rec(p, r, depth + 1)
    rec(root, b".", 0)
    return out


def _groups(w: dict) -> dict:
    """rel -> the sorted paths of the same tree that share its inode (itself included)."""
    by = {}
    for rel, st in w.items():
        if stat.S_ISREG(st.st_mode):
            by.setdefault((st.st_dev, st.st_ino), []).append(rel)
    return {rel: sorted(g) for g in by.values() for rel in g}


def _esc(raw: bytes) -> bytes:
    out = bytearray()
    for c in raw:
        out += {0x5C: b"\\\\", 0x09: b"\\t", 0x0A: b"\\n"}.get(c, b"\\x%02x" % c if c < 0x20 else bytes([c]))
    return bytes(out)


def _identity(table) -> dict:
    t = _orc.read_table(table)
    return {rel: (size, ino, ct) for (rel, size, _first), (ino, ct) in zip(t["entries"], t["identity"])}


def expected(layer, snap, bb, flags=0, layer_table=None):
    """(report bytes, counters) of vmig_compare_snapshot(layer, layer_table, snap, <snap's table>), by include/vmig.h."""
    vm = _vm
    skip, ns, nometa = flags & vm.F_SKIP_HIDDEN_TOPDIRS, flags & vm.F_MTIME_NS, flags & vm.F_NO_METADATA
    L, S = _walk(layer, skip), _walk(snap, skip)
    gl, gs = _groups(L), _groups(S)
    rec = _identity(layer_table) if layer_table else {}
    lroot, sroot = os.fsencode(os.fspath(layer)), os.fsencode(os.fspath(snap))
    c = dict.fromkeys(COUNTERS, 0)
    read = {}
    lines = []
    nb = lambda n: -(-n // bb)
    mt = lambda st: (b"%d.%09d" % divmod(st.st_mtime_ns, 10**9)) if ns else b"%d" % (st.st_mtime_ns // 10**9)
    for rel in sorted(set(L) | set(S)):
        e = _esc(rel)
        if rel not in S:
            lines.append(b"added\t%s\t-\t-\t-\n" % e)
            c["paths_added"] += 1
            continue
        if rel not in L:
            lines.append(b"removed\t%s\t-\t-\t-\n" % e)
            c["paths_removed"] += 1
            if stat.S_ISREG(S[rel].st_mode):
                c["bytes_restore"] += S[rel].st_size
            continue
        l, s = L[rel], S[rel]
        mine = []
        lt, st_ = stat.S_IFMT(l.st_mode), stat.S_IFMT(s.st_mode)
        if lt != st_:
            mine.append(b"type\t%s\t-\t%s\t%s\n" % (e, TYPE[lt], TYPE[st_]))
            if st_ == stat.S_IFREG:
                c["bytes_restore"] += s.st_size
        elif rel != b".":
            if lt == stat.S_IFREG:
                nl, nsb = nb(l.st_size), nb(s.st_size)
                if nl and nsb:
                    r_ = rec.get(rel)
                    if (l.st_dev, l.st_ino, l.st_size) == (s.st_dev, s.st_ino, s.st_size):
                        c["files_shared"] += 1
                    elif r_ and r_[1] != 0 and (r_[0], r_[1], r_[2]) == (l.st_size, l.st_ino, l.st_ctime_ns):
                        c["files_trusted"] += 1
                    else:
                        read[(l.st_dev, l.st_ino)] = l.st_size
                lh = [int(h) for h in _orc.hash_file(os.path.join(lroot, rel), bb)]
                sh = [int(h) for h in _orc.hash_file(os.path.join(sroot, rel), bb)]
                changed = False
                if l.st_size != s.st_size:
                    mine.append(b"resized\t%s\t-\t%d\t%d\n" % (e, l.st_size, s.st_size))
                    changed = True
                for r in range(nsb):
                    slen = min(bb, s.st_size - r * bb)
                    differs = r >= nl
                    if not differs:
                        differs = min(bb, l.st_size - r * bb) != slen or lh[r] != sh[r]
                        if differs:
                            mine.append(b"block\t%s\t%d\t%016x\t%016x\n" % (e, r, lh[r], sh[r]))
                            c["blocks_changed"] += 1
                            changed = True
                    if differs:
                        c["bytes_restore"] += slen
                c["files_changed"] += changed
                if gl[rel] != gs[rel]:
                    first = lambda g: _esc(g[0]) if len(g) > 1 else b"-"
                    mine.append(b"hardlink\t%s\t-\t%s\t%s\n" % (e, first(gl[rel]), first(gs[rel])))
            elif lt == stat.S_IFLNK:
                a, b = os.readlink(os.path.join(lroot, rel)), os.readlink(os.path.join(sroot, rel))
                if a != b:
                    mine.append(b"target\t%s\t-\t%s\t%s\n" % (e, _esc(a), _esc(b)))
            elif lt in (stat.S_IFCHR, stat.S_IFBLK) and l.st_rdev != s.st_rdev:
                mine.append(b"rdev\t%s\t-\t%d:%d\t%d:%d\n" % (e, os.major(l.st_rdev), os.minor(l.st_rdev), os.major(s.st_rdev),
                                                              os.minor(s.st_rdev)))
        if lt == st_ and not nometa:
            if stat.S_IMODE(l.st_mode) != stat.S_IMODE(s.st_mode):
                mine.append(b"mode\t%s\t-\t%04o\t%04o\n" % (e, stat.S_IMODE(l.st_mode), stat.S_IMODE(s.st_mode)))
            if (l.st_uid, l.st_gid) != (s.st_uid, s.st_gid):
                mine.append(b"owner\t%s\t-\t%d:%d\t%d:%d\n" % (e, l.st_uid, l.st_gid, s.st_uid, s.st_gid))
            if mt(l) != mt(s):
                mine.append(b"mtime\t%s\t-\t%s\t%s\n" % (e, mt(l), mt(s)))
        c["paths_changed"] += bool(mine)
        lines += mine
    c["files_read"], c["bytes_read"] = len(read), sum(read.values())
    return b"".join(lines), c


_vm = _orc = None


@pytest.fixture(autouse=True)
def _oracle_modules(vm, orc):
    global _vm, _orc
    _vm, _orc = vm, orc


def check(vm, layer, snap, table, report, bb, flags=0, layer_table=None, lanes=1):
    """One compare held to the oracle: report and counters; returns the call's result."""
    r = vm.compare_snapshot(layer, snap, table, report, layer_table, flags=flags, block_bytes=bb, lanes_per_gpu=lanes)
    want, c = expected(layer, snap, bb, flags, layer_table)
    got = Path(report).read_bytes()
    assert got == want, (flags, layer_table, got.decode(errors="replace"), want.decode(errors="replace"))
    assert {k: r[k] for k in COUNTERS} == c, (flags, layer_table, r, c)
    assert r["stats"]["bytes_h2d"] == r["bytes_read"] and r["stats"]["bytes_total"] == r["bytes_read"]
    return r


# ------------------------------------------------------------------------------------------ trees
def _flip(p: Path, off: int, keep_mtime: bool = True):
    st = os.stat(p)
    with open(p, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x5A]))
    if keep_mtime:
        os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns))


PAIRS = [(a, b) for a in lm.KINDS for b in lm.KINDS if a != b]
MB_FILES = ("first", "mid", "last", "grow", "shrink", "tozero", "fromzero")


def _source(orc, src: Path, bb: int, hardlinks: bool = True):
    make_rich_tree(src, orc)
    if not hardlinks:
        os.unlink(src / "sub" / "hard1")
        os.unlink(src / "a_hard2")
    (src / "k").mkdir()
    for i, (a, _b) in enumerate(PAIRS):
        if hardlinks or a != "hardlink":
            lm.make_kind(src, f"k/{i}", a, i)
    (src / "mb").mkdir()
    for i, n in enumerate(MB_FILES):
        (src / "mb" / n).write_bytes(b"" if n == "fromzero" else lm.data(40 + i, 3 * bb + 100))
    (src / "hl").mkdir()
    for n in ("x", "y", "p"):
        (src / "hl" / n).write_bytes(b"same content")
    if hardlinks:
        os.link(src / "hl" / "p", src / "hl" / "q")
    (src / "aw").mkdir()
    for i in range(len(lm.NAME_POOL)):
        (src / "aw" / lm.awkward(i, room=8)).write_bytes(lm.data(60 + i, 3000 + i))


def _mutate(layer: Path, bb: int):
    for i, (_a, b) in enumerate(PAIRS):                                   # every kind change
        lm.make_kind(layer, f"k/{i}", b, i + 100)
    mb = layer / "mb"
    _flip(mb / "first", 0)                                                # first, middle and short last block
    _flip(mb / "mid", bb + 5)
    _flip(mb / "last", 3 * bb + 99)
    with open(mb / "grow", "ab") as f:
        f.write(lm.data(70, bb))
    os.truncate(mb / "shrink", bb + 10)
    os.truncate(mb / "tozero", 0)
    (mb / "fromzero").write_bytes(lm.data(71, 2 * bb + 3))
    (layer / "newdir" / "a").mkdir(parents=True)                          # adds and removes of files and subtrees
    (layer / "newdir" / "a" / "b").write_bytes(b"new")
    (layer / "newfile").write_bytes(b"new file")
    shutil.rmtree(layer / "sub")
    os.unlink(layer / "exact.bin")
    os.unlink(layer / "lnk")                                              # symlink retarget
    os.symlink("zeros.bin", layer / "lnk")
    os.chmod(layer / "zeros.bin", 0o600)                                  # chmod; chown where run as root
    if os.geteuid() == 0:
        os.chown(layer / "big.bin", 4242, 4343)
        os.unlink(layer / "whiteout")
        os.mknod(layer / "whiteout", 0o020000 | 0o644, os.makedev(7, 9))
    st = os.stat(layer / "empty")                                         # a sub-second mtime change
    os.utime(layer / "empty", ns=(st.st_atime_ns, st.st_mtime_ns // 10**9 * 10**9 + 5))
    os.unlink(layer / "hl" / "y")                                         # a hard link made, one broken
    os.link(layer / "hl" / "x", layer / "hl" / "y")
    os.unlink(layer / "hl" / "q")
    (layer / "hl" / "q").write_bytes(b"same content")
    names = sorted(os.listdir(layer / "aw"))                              # awkward names: edit, remove, add
    for i, n in enumerate(names):
        if i % 3 == 0:
            os.unlink(layer / "aw" / n)
        elif i % 3 == 1:
            _flip(layer / "aw" / n, 10)
    (layer / "aw" / (lm.NAME_POOL[1] + "+added")).write_bytes(b"x")
    (layer / ".hidden_dir" / "inner").write_bytes(b"hidden edit")         # seen only without VMIG_F_SKIP_HIDDEN_TOPDIRS
    (layer / ".hidden_dir" / "new").write_bytes(b"hidden add")


def _setup(vm, orc, root: Path, bb: int, lanes: int = 1, hardlinks: bool = True):
    """root/src, its snapshot root/snap (root/snap.vmig) and root/layer, a restore of it (table root/layer.vmig)."""
    src, snap, layer = root / "src", root / "snap", root / "layer"
    src.mkdir()
    _source(orc, src, bb, hardlinks)
    snap.mkdir()
    layer.mkdir()
    vm.snapshot_tree(src, snap, None, None, root / "snap.vmig", block_bytes=bb, lanes_per_gpu=lanes)
    vm.restore_tree(snap, root / "snap.vmig", layer, None, root / "layer.vmig", block_bytes=bb, lanes_per_gpu=lanes)
    return src, snap, root / "snap.vmig", layer, root / "layer.vmig"


# ------------------------------------------------------------------------------------------ 1. a restored layer
def test_restored_layer_compares_empty(vm, orc, shm_tmp):
    bb = 1 << 20
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, hardlinks=False)
    report = shm_tmp / "cmp.txt"
    r = check(vm, layer, snap, t, report, bb)
    assert report.read_bytes() == b"" and r["bytes_read"] > 0 and r["paths_changed"] == 0 and r["bytes_restore"] == 0
    r = check(vm, layer, snap, t, report, bb, layer_table=lt)
    assert report.read_bytes() == b"" and r["files_read"] == 0 and r["stats"]["bytes_h2d"] == 0 and r["files_trusted"] > 0


# ------------------------------------------------------------------------------------------ 2. a mutated layer
@pytest.mark.parametrize("bb,lanes", [(4096, 1), ((1 << 20) + 4096, 3), (4 << 20, 1), (4 << 20, 3)])
def test_mutated_layer_matches_oracle(vm, orc, shm_tmp, bb, lanes):
    src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb, lanes)
    _mutate(layer, bb)
    report = shm_tmp / "cmp.txt"
    for flags in (0, vm.F_MTIME_NS, vm.F_NO_METADATA, vm.F_DIRECT_IO):
        r = check(vm, layer, snap, t, report, bb, flags, lanes=lanes)
    kinds = {f["kind"] for f in vm.parse_compare_report(report)}
    want_kinds = set(vm.COMPARE_KINDS) - ({"owner", "rdev"} if os.geteuid() else set())
    assert kinds == want_kinds, kinds
    ns = vm.parse_compare_report(report)
    check(vm, layer, snap, t, report, bb, vm.F_MTIME_NS, lanes=lanes)
    assert any(f["kind"] == "mtime" and f["path"] == "empty" for f in vm.parse_compare_report(report))
    assert not any(f["kind"] == "mtime" and f["path"] == "empty" for f in ns)
    # the hidden top-level directory is not walked on either side; the snapshot is taken with the same flag
    snap_h = shm_tmp / "snap_h"
    snap_h.mkdir()
    vm.snapshot_tree(src, snap_h, None, None, shm_tmp / "snap_h.vmig", flags=vm.F_SKIP_HIDDEN_TOPDIRS, block_bytes=bb)
    check(vm, layer, snap_h, shm_tmp / "snap_h.vmig", report, bb, vm.F_SKIP_HIDDEN_TOPDIRS, lanes=lanes)
    assert not any(f["path"].startswith(".hidden_dir") for f in vm.parse_compare_report(report))


# ------------------------------------------------------------------------------------------ 3. the layer's own table
def test_layer_table_reads_only_moved_identities(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    _flip(layer / "big.bin", 3 * bb + 1, keep_mtime=False)               # an edit
    _flip(layer / "mb" / "mid", bb + 5, keep_mtime=True)                 # an edit that put the mtime back
    os.chmod(layer / "mb" / "last", 0o600)                               # metadata only: the ctime moves too
    report, report_t = shm_tmp / "cmp.txt", shm_tmp / "cmp_t.txt"
    full = check(vm, layer, snap, t, report, bb)
    r = check(vm, layer, snap, t, report_t, bb, layer_table=lt)
    assert report.read_bytes() == report_t.read_bytes() and report.read_bytes() != b""
    # read: the three files whose identity moved, and the hard-linked paths, which a table records without identity
    assert 3 <= r["files_read"] < full["files_read"] and r["files_trusted"] > 0
    assert {f["path"] for f in vm.parse_compare_report(report_t) if f["kind"] == "block"} == {"big.bin", "sub/hard1", "mb/mid"}


# ------------------------------------------------------------------------------------------ 4. versions of one store
def test_versions_of_an_incremental_store(vm, orc, shm_tmp):
    bb, n = 65536, 4
    src = shm_tmp / "src"
    lm.build_layer(src, orc, bb, make_rich_tree)
    ops = [[]] + lm.script(21, n, bb)
    V = []
    for k in range(n + 1):
        lm.apply(src, ops[k])
        d, tab = shm_tmp / f"v{k}", shm_tmp / f"v{k}.vmig"
        d.mkdir()
        base = V[-1] if V else (None, None)
        vm.snapshot_tree(src, d, base[0], base[1], tab, block_bytes=bb)
        V.append((d, tab))
    report = shm_tmp / "cmp.txt"
    for j in range(n + 1):
        for k in (j - 1, j + 1, n):
            if 0 <= k <= n and k != j:
                r = check(vm, V[k][0], V[j][0], V[j][1], report, bb)
                assert r["files_shared"] > 0 or abs(k - j) > 1, (k, j, r)
    r = check(vm, V[n][0], V[n][0], V[n][1], report, bb)                  # a version against itself reads nothing
    assert report.read_bytes() == b"" and r["files_read"] == 0 and r["files_shared"] > 0


# ------------------------------------------------------------------------------------------ 5. preview equals effect
def test_preview_equals_effect(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    _mutate(layer, bb)
    report = shm_tmp / "cmp.txt"
    check(vm, layer, snap, t, report, bb)
    preview = {f["path"] for f in vm.parse_compare_report(report)}
    copy = shm_tmp / "copy"
    lm.freeze(layer, copy)
    before = orc.tree_manifest(copy)
    vm.restore_tree(snap, t, copy, flags=vm.F_PRUNE, block_bytes=bb)
    after = orc.tree_manifest(copy)
    effect = {rel for rel in set(before) | set(after) if before.get(rel) != after.get(rel)}
    assert preview == effect, (sorted(preview - effect), sorted(effect - preview))
    check(vm, copy, snap, t, report, bb)
    assert report.read_bytes() == b""


# ------------------------------------------------------------------------------------------ 6. a damaged snapshot
def test_snapshot_that_does_not_match_its_table_is_refused(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    report = shm_tmp / "cmp.txt"
    for name, damage, path in (("missing", lambda d: os.unlink(d / "mb" / "mid"), "mb/mid"),
                               ("extra", lambda d: (d / "mb" / "zz").write_bytes(b"x"), "mb/zz"),
                               ("resized", lambda d: open(d / "mb" / "last", "ab").write(b"x"), "mb/last")):
        bad = shm_tmp / f"snap_{name}"
        lm.freeze(snap, bad)
        damage(bad)
        with pytest.raises(vm.VmigError) as ei:
            vm.compare_snapshot(layer, bad, t, report, block_bytes=bb)
        assert ei.value.code == vm.VMIG_ECORRUPT and path in str(ei.value) and f"({name})" in str(ei.value), ei.value
        assert not any(n.startswith("cmp.txt") for n in os.listdir(shm_tmp))


# ------------------------------------------------------------------------------------------ 7. read-only
def _lstat_all(*roots):
    out = {}
    for root in roots:
        root = os.fsencode(os.fspath(root))
        out[root] = (os.lstat(root).st_ino, os.lstat(root).st_ctime_ns, os.lstat(root).st_mtime_ns)
        for dp, dns, fns in os.walk(root):
            for n in dns + fns:
                s = os.lstat(os.path.join(dp, n))
                out[os.path.join(dp, n)] = (s.st_ino, s.st_ctime_ns, s.st_mtime_ns)
    return out


def test_compare_is_read_only(vm, orc, shm_tmp):
    bb = 65536
    _src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    _mutate(layer, bb)
    before = _lstat_all(snap, layer, t, lt)
    listing = sorted(os.listdir(shm_tmp))
    report = shm_tmp / "cmp.txt"
    check(vm, layer, snap, t, report, bb, layer_table=lt)
    check(vm, layer, snap, t, report, bb, vm.F_DIRECT_IO)
    assert _lstat_all(snap, layer, t, lt) == before
    assert sorted(os.listdir(shm_tmp)) == sorted(listing + ["cmp.txt"])


# ------------------------------------------------------------------------------------------ 8. cancel and phases
def test_cancel_half_way_then_succeed(vm, orc, shm_tmp):
    bb = 4 << 20
    src, snap = shm_tmp / "src", shm_tmp / "snap"
    src.mkdir()
    chunk = lm.data(3, 128 * MiB)
    for i in range(16):
        (src / f"f{i:02d}").write_bytes(chunk)
    snap.mkdir()
    vm.snapshot_tree(src, snap, None, None, shm_tmp / "snap.vmig", block_bytes=bb)
    report = shm_tmp / "cmp.txt"
    with vm.Ctl() as c:
        returned = threading.Event()

        def canceller():
            while not returned.is_set():
                p = c.progress()
                if p["bytes_total"] and p["bytes_hashed"] >= p["bytes_total"] // 2:
                    c.cancel()
                    return
                time.sleep(0.0005)
        th = threading.Thread(target=canceller)
        th.start()
        try:
            with pytest.raises(vm.VmigError) as ei:
                vm.compare_snapshot(src, snap, shm_tmp / "snap.vmig", report, block_bytes=bb, ctl=c)
        finally:
            returned.set()
            th.join()
        assert ei.value.code == vm.VMIG_ECANCELED, ei.value
    assert not any(n.startswith("cmp.txt") for n in os.listdir(shm_tmp))
    with vm.Ctl() as c:
        seen, done = [], threading.Event()

        def watch():
            while not done.is_set():
                ph = c.progress()["phase_name"]
                if not seen or seen[-1] != ph:
                    seen.append(ph)
                time.sleep(0.0002)
        th = threading.Thread(target=watch)
        th.start()
        try:
            r = vm.compare_snapshot(src, snap, shm_tmp / "snap.vmig", report, block_bytes=bb, ctl=c)
        finally:
            done.set()
            th.join()
        seen.append(c.progress()["phase_name"])
    order = ["IDLE", "WALK", "DATA", "DONE"]
    assert [order.index(p) for p in seen] == sorted(order.index(p) for p in seen) and seen[-1] == "DONE", seen
    assert "DATA" in seen and report.read_bytes() == b"" and r["bytes_read"] == 16 * 128 * MiB


# ------------------------------------------------------------------------------------------ 9. alongside other calls
def test_compare_alongside_a_migration_and_a_snapshot(vm, orc, shm_tmp):
    bb = 1 << 20
    src, snap, t, layer, lt = _setup(vm, orc, shm_tmp, bb)
    _mutate(layer, bb)
    big = shm_tmp / "big"
    big.mkdir()
    for i in range(6):
        (big / f"f{i}").write_bytes(lm.data(80 + i, 48 * MiB + i))
    (shm_tmp / "mig").mkdir()
    (shm_tmp / "inc").mkdir()
    (src / "edited").write_bytes(b"for the increment")
    want, want_c = expected(layer, snap, bb)
    errs, out = [], {}

    def run(name, fn):
        try:
            out[name] = fn()
        except Exception as e:                       # noqa: BLE001 -- reported below
            errs.append((name, e))
    calls = {
        "compare": lambda: vm.compare_snapshot(layer, snap, t, shm_tmp / "cmp.txt", block_bytes=bb, lanes_per_gpu=2),
        "migrate": lambda: vm.migrate_tree(big, shm_tmp / "mig", block_bytes=bb),
        "snapshot": lambda: vm.snapshot_tree(src, shm_tmp / "inc", snap, t, shm_tmp / "inc.vmig", block_bytes=bb),
    }
    ths = [threading.Thread(target=run, args=kv) for kv in calls.items()]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errs, errs
    assert (shm_tmp / "cmp.txt").read_bytes() == want and {k: out["compare"][k] for k in COUNTERS} == want_c
    assert orc.compare_trees(big, shm_tmp / "mig") == []
    full = shm_tmp / "full"                          # the increment holds what a full snapshot taken now holds
    full.mkdir()
    vm.snapshot_tree(src, full, None, None, shm_tmp / "full.vmig", block_bytes=bb)
    assert lm.diff_manifests(lm.tree_in_itself(orc, full), lm.tree_in_itself(orc, shm_tmp / "inc")) == []
    assert out["snapshot"]["files_linked"] > 0


# ------------------------------------------------------------------------------------------ 10. the hand-off mirror
def test_compare_with_version_after_a_handoff(vm, orc, shm_tmp):
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {n: shm_tmp / f"upper_{n}" for n in ("rs-1", "rs-2", "rs-3")}
    ups["rs-1"].mkdir()
    ups["rs-3"].mkdir()
    make_rich_tree(ups["rs-1"], orc)
    os.unlink(ups["rs-1"] / "sub" / "hard1")            # hard-linked paths carry no identity in a table: always read
    os.unlink(ups["rs-1"] / "a_hard2")
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersion("rs-1")
        lm.freeze(ups["rs-1"], ups["rs-2"])              # the running container, then its Patch successor rs-3
        st1 = os.stat(ups["rs-1"])
        os.chmod(ups["rs-2"], stat.S_IMODE(st1.st_mode))
        os.utime(ups["rs-2"], ns=(st1.st_atime_ns, st1.st_mtime_ns))
        ho.HandoffCopy("rs-2", "rs-3", pause=lambda n: None, resume=lambda n: None)
        assert not ho.snapshotPaths("rs-3")[0].exists() and ho.snapshotPaths("rs-3")[1].exists()
        _flip(ups["rs-3"] / "exact.bin", 5, keep_mtime=True)   # the tenant's edit
        report = shm_tmp / "cmp.txt"
        r = ho.CompareWithVersion("rs-1", "rs-3", report)
        data, table = ho.snapshotPaths("rs-1")
        want, c = expected(ups["rs-3"], data, vm.BLOCK_BYTES, 0, ho.snapshotPaths("rs-3")[1])
        assert report.read_bytes() == want and {k: r[k] for k in COUNTERS} == c
        assert [(f["kind"], f["path"], f["block"]) for f in vm.parse_compare_report(report)] == [("block", "exact.bin", 0)]
        assert r["files_read"] == 1 and r["bytes_read"] == 4 << 20
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
