"""vmig_scrub_store on the GPU (-m gpu): one pass over a snapshot store built with vmig_snapshot_tree (v1 full, later
versions incremental with a rename, one changed file and 30 % changed blocks, over make_rich_tree plus awkward names).

The expected verdict of every version is what a hash-only restore of it returns; the expected hash of every block is the
oracle's (C XXH64 over the file on disk), the wanted one the table's own, read here from the documented file format."""
import hashlib
import os
import re
import struct
import subprocess
import threading
import time
from pathlib import Path

import numpy as np
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


# ------------------------------------------------------------------------------------------ store
def _flip(p: Path, off: int, keep_mtime: bool = False):
    st = os.stat(p)
    with open(p, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x5A]))
    if keep_mtime:
        os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns))


def _source(orc, src: Path):
    make_rich_tree(src, orc)
    d = src / "data"
    d.mkdir()
    (d / "keep.bin").write_bytes(orc.splitmix_bytes(31, 2 * BB + 100).tobytes())
    (d / "g1.bin").write_bytes(orc.splitmix_bytes(32, 3 * BB + 5).tobytes())
    (d / "g2.bin").write_bytes(orc.splitmix_bytes(33, 10 * BB).tobytes())
    (d / "g3.bin").write_bytes(orc.splitmix_bytes(34, 2 * BB).tobytes())
    for name in ("tab\tname.bin", "nl\nname.bin", "back\\slash.bin", "ctl\x01char.bin"):
        (src / name).write_bytes(orc.splitmix_bytes(len(name), BB + 17).tobytes())


def build_store(vm, orc, root: Path, n_versions: int = 4, **kw):
    """root/src and its snapshots root/v1..vN with tables root/vK.vmig: v2 renames a file, v3 changes one block of one
    file, v4 changes 30 % of the blocks of another, v5 changes the first file again.  Returns [(dir, table)]."""
    src = root / "src"
    src.mkdir(parents=True)
    _source(orc, src)
    pairs = []
    for k in range(1, n_versions + 1):
        if k == 2:
            (src / "moved").mkdir()
            os.rename(src / "data" / "g3.bin", src / "moved" / "g3.bin")
        elif k == 3:
            _flip(src / "data" / "g1.bin", BB + 7)
        elif k == 4:
            for b in (1, 4, 8):
                _flip(src / "data" / "g2.bin", b * BB + 3)
        elif k == 5:
            _flip(src / "data" / "g1.bin", 11)
        d, t = root / f"v{k}", root / f"v{k}.vmig"
        d.mkdir()
        base = pairs[-1] if pairs else (None, None)
        vm.snapshot_tree(src, d, base[0], base[1], t, **kw)
        pairs.append((d, t))
    return pairs


def read_table(path):
    """{rel: (size, [hash per block], ino, ctime_ns)} of a VMIGBT02 block table (include/vmig.h)."""
    raw = Path(path).read_bytes()
    assert raw[:8] == b"VMIGBT02"
    bb, _algo, nf, nb = struct.unpack_from("<IIQQ", raw, 8)
    off, files = 32, []
    for _ in range(nf):
        (pl,) = struct.unpack_from("<I", raw, off)
        rel = os.fsdecode(raw[off + 4:off + 4 + pl])
        off += 4 + pl
        size, fb, ino, ct = struct.unpack_from("<QQQq", raw, off)
        off += 32
        files.append((rel, size, fb, ino, ct))
    hashes = np.frombuffer(raw, dtype="<u8", count=nb, offset=off)
    return {rel: (size, [int(h) for h in hashes[fb:fb + (size + bb - 1) // bb]], ino, ct) for rel, size, fb, ino, ct in files}


def regular_files(root: Path) -> dict:
    out = {}
    for dp, _dns, fns in os.walk(root):
        for n in fns:
            p = os.path.join(dp, n)
            st = os.lstat(p)
            if os.path.isfile(p) and not os.path.islink(p):
                out[os.path.relpath(p, root)] = st
    return out


def restore_verdict(vm, d, t):
    try:
        vm.restore_tree(d, t, None, flags=vm.F_HASH_ONLY)
        return vm.VMIG_OK, ""
    except vm.VmigError as e:
        return e.code, vm.last_error()


def restore_finding(code, msg, vm):
    """(kind, path, block) of the first difference a hash-only restore reports."""
    if code == vm.VMIG_ETABLE:
        return ("table", ".", None)
    for kind, rx in (("extra", r"(.*) is in the snapshot but not in its block table \(extra\)"),
                     ("missing", r"(.*) is in the block table but not in the snapshot \(missing\)"),
                     ("resized", r"(.*) is \d+ bytes in the snapshot, \d+ in its block table \(resized\)"),
                     ("hardlink", r"(.*) block (\d+) \(a hard link to .*\) hashes [0-9a-f]{16}, its block table says [0-9a-f]{16}"),
                     ("block", r"(.*) block (\d+) hashes [0-9a-f]{16}, its block table says [0-9a-f]{16}")):
        m = re.fullmatch(rx, msg, flags=re.S)
        if m:
            return (kind, m.group(1), int(m.group(2)) if m.lastindex >= 2 else None)
    raise AssertionError(f"unparsed restore error: {msg!r}")


def check_against_restore_and_oracle(vm, orc, pairs, r):
    assert len(r["verdicts"]) == len(pairs)
    for i, (d, t) in enumerate(pairs):
        code, msg = restore_verdict(vm, d, t)
        assert r["verdicts"][i] == code, (i, r["verdicts"][i], code, msg)
        mine = [f for f in r["findings"] if f["version"] == i]
        assert (code == vm.VMIG_OK) == (not mine), (i, mine)
        if code != vm.VMIG_OK:
            assert restore_finding(code, msg, vm) in [(f["kind"], f["path"], f["block"]) for f in mine], (msg, mine)
        if code == vm.VMIG_ETABLE:
            continue
        table, walk = read_table(t), regular_files(d)
        flagged = {(f["path"], f["block"]) for f in mine if f["kind"] in ("block", "hardlink")}
        for f in mine:
            if f["kind"] in ("block", "hardlink"):
                assert f["got"] == int(orc.hash_file(d / f["path"])[f["block"]]), f
                assert f["want"] == table[f["path"]][1][f["block"]], f
        for rel, (size, hashes, _ino, _ct) in table.items():          # nothing damaged goes unflagged
            if rel not in walk or walk[rel].st_size != size:
                continue
            got = orc.hash_file(d / rel) if size else []
            for b, h in enumerate(hashes):
                assert (int(got[b]) != h) == ((rel, b) in flagged), (i, rel, b)


def store_state(root: Path) -> dict:
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            s = os.lstat(p)
            body = hashlib.sha256(Path(p).read_bytes()).hexdigest() if os.path.isfile(p) and not os.path.islink(p) else None
            out[p] = (s.st_ino, s.st_nlink, s.st_mode, s.st_size, s.st_mtime_ns, s.st_ctime_ns, body)
    return out


# ------------------------------------------------------------------------------------------ 1. clean store
def test_clean_store_reads_each_inode_once(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp)
    report = shm_tmp / "scrub.txt"
    r = vm.scrub_store(pairs, report)
    assert r["verdicts"] == [vm.VMIG_OK] * 4 and r["findings"] == [] and report.read_bytes() == b""
    distinct, referenced = {}, 0
    for d, _ in pairs:
        for st in regular_files(d).values():
            distinct[(st.st_dev, st.st_ino)] = st.st_size
            referenced += st.st_size
    assert r["bytes_unique"] == sum(distinct.values()) < r["bytes_referenced"] == referenced, r
    assert r["stats"]["bytes_h2d"] == r["bytes_unique"] == r["stats"]["bytes_total"]
    assert r["versions"] == 4 and r["versions_damaged"] == r["files_damaged"] == r["blocks_damaged"] == r["files_unreadable"] == 0
    check_against_restore_and_oracle(vm, orc, pairs, r)


# ------------------------------------------------------------------------------------------ 2. agreement with restore
def damage(pairs):
    """Every kind of damage a store meets; version 5 loses its table."""
    (v1, _), (v2, _), (v3, _), (v4, _), (_, t5) = pairs
    assert os.stat(v1 / "data" / "keep.bin").st_nlink == 5            # one inode shared by every version
    _flip(v1 / "data" / "keep.bin", BB + 9, keep_mtime=True)
    assert os.stat(v4 / "data" / "g2.bin").st_nlink == 2                # written new in v4, linked by v5 only
    _flip(v4 / "data" / "g2.bin", 3 * BB + 1)
    (v1 / "extra.txt").write_bytes(b"not in the table\n")
    os.truncate(v2 / "big.bin", 5 * MiB)                                # shared with v2/sub/hard1 only
    (v2 / ".dotfile").unlink()
    os.mkfifo(v2 / ".dotfile")
    (v3 / "moved" / "g3.bin").unlink()
    t5.unlink()


def test_verdicts_and_findings_agree_with_restore(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp, n_versions=5)
    damage(pairs)
    r = vm.scrub_store(pairs, shm_tmp / "scrub.txt")
    C, T = vm.VMIG_ECORRUPT, vm.VMIG_ETABLE
    assert r["verdicts"] == [C, C, C, C, T], r["verdicts"]
    kinds = {(f["version"], f["kind"], f["path"]) for f in r["findings"]}
    for want in [(0, "extra", "extra.txt"), (1, "resized", "big.bin"), (1, "resized", "sub/hard1"), (1, "missing", ".dotfile"),
                 (2, "missing", "moved/g3.bin"), (3, "block", "data/g2.bin"), (4, "table", ".")]:
        assert want in kinds, (want, kinds)
    for v in range(4):
        assert (v, "block", "data/keep.bin") in kinds
    assert r["versions_damaged"] == 5 and r["files_unreadable"] == 0
    check_against_restore_and_oracle(vm, orc, pairs, r)


def test_awkward_names_round_trip_through_the_report(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp, n_versions=2)
    for name in ("tab\tname.bin", "nl\nname.bin", "back\\slash.bin", "ctl\x01char.bin"):
        _flip(pairs[1][0] / name, 5, keep_mtime=True)                  # linked: both versions see it
    report = shm_tmp / "scrub.txt"
    r = vm.scrub_store(pairs, report)
    lines = report.read_bytes().split(b"\n")
    assert lines[-1] == b"" and len(lines) - 1 == len(r["findings"]) == 8
    assert all(ln.count(b"\t") == 5 for ln in lines[:-1])
    assert {f["path"] for f in r["findings"]} == {"tab\tname.bin", "nl\nname.bin", "back\\slash.bin", "ctl\x01char.bin"}
    keys = [(f["version"], os.fsencode(f["path"]), f["block"]) for f in r["findings"]]
    assert keys == sorted(keys)                                          # by version, then the raw path bytes, then block
    check_against_restore_and_oracle(vm, orc, pairs, r)


# ------------------------------------------------------------------------------------------ 3. blast radius
def test_one_flipped_byte_in_a_shared_inode_marks_every_version_that_links_it(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp)
    target = pairs[0][0] / "exact.bin"
    assert os.stat(target).st_nlink == 4
    _flip(target, 12345, keep_mtime=True)
    r = vm.scrub_store(pairs, shm_tmp / "scrub.txt")
    assert r["verdicts"] == [vm.VMIG_ECORRUPT] * 4
    assert [(f["version"], f["kind"], f["path"], f["block"]) for f in r["findings"]] == [(v, "block", "exact.bin", 0) for v in range(4)]
    assert r["blocks_damaged"] == 1 and r["files_damaged"] == 4 and r["versions_damaged"] == 4
    check_against_restore_and_oracle(vm, orc, pairs, r)


# ------------------------------------------------------------------------------------------ 4. read-only
def test_scrub_writes_nothing_and_keeps_every_identity(vm, orc, shm_tmp):
    pairs = build_store(vm, orc, shm_tmp)
    before = store_state(shm_tmp)
    r = vm.scrub_store(pairs, None)
    assert r["verdicts"] == [vm.VMIG_OK] * 4
    assert store_state(shm_tmp) == before
    # the next increment still trusts and links every unchanged file of the newest version
    src = shm_tmp / "src"
    unchanged = sum(1 for st in regular_files(src).values() if st.st_nlink == 1 and st.st_size > 0)
    v5 = shm_tmp / "v5"
    v5.mkdir()
    st = vm.snapshot_tree(src, v5, pairs[-1][0], pairs[-1][1], shm_tmp / "v5.vmig")
    assert st["files_linked"] == unchanged and st["bytes_written"] == 0, st


# ------------------------------------------------------------------------------------------ 5. lanes and O_DIRECT
def _disk_dir(tmp_path: Path) -> Path:
    fs = subprocess.run(["stat", "-f", "-c", "%T", str(tmp_path)], capture_output=True, text=True).stdout.strip()
    if fs in ("tmpfs", "ramfs"):
        pytest.skip(f"needs a disk-backed temporary directory for O_DIRECT ({tmp_path} is {fs})")
    probe = tmp_path / "odirect_probe"
    try:
        fd = os.open(probe, os.O_WRONLY | os.O_CREAT | os.O_DIRECT, 0o600)
        os.close(fd)
    except OSError as e:
        pytest.skip(f"the filesystem of {tmp_path} refuses O_DIRECT: {e}")
    probe.unlink()
    return tmp_path


@pytest.mark.parametrize("mode", ["3lanes", "direct"])
def test_same_report_with_three_lanes_and_direct_io(vm, orc, shm_tmp, tmp_path, mode):
    root = _disk_dir(tmp_path) if mode == "direct" else shm_tmp
    pairs = build_store(vm, orc, root, n_versions=5)
    damage(pairs)
    base = vm.scrub_store(pairs, root / "plain.txt")
    kw = {"lanes_per_gpu": 3} if mode == "3lanes" else {"flags": vm.F_DIRECT_IO}
    other = vm.scrub_store(pairs, root / "other.txt", **kw)
    assert other["verdicts"] == base["verdicts"]
    assert (root / "other.txt").read_bytes() == (root / "plain.txt").read_bytes()
    if mode == "3lanes":
        assert other["stats"]["lanes_used"] == 3
    else:
        assert other["stats"]["files_direct"] > 0


# ------------------------------------------------------------------------------------------ 6. cancellation
class Canceller(threading.Thread):
    """Polls ctl.progress() every 0.5 ms and cancels once pred(progress) holds (as tests/test_cancel.py does)."""

    def __init__(self, ctl, pred):
        super().__init__(daemon=True)
        self.ctl, self.pred, self.fired, self.done = ctl, pred, False, threading.Event()

    def run(self):
        while not self.done.is_set():
            if self.pred(self.ctl.progress()):
                self.fired = True
                self.ctl.cancel()
                return
            time.sleep(0.0005)


def _threads():
    return len(os.listdir("/proc/self/task"))


def _fds():
    return len(os.listdir("/proc/self/fd"))


def test_cancel_at_half_leaves_no_report(vm, orc, shm_tmp):
    src, v1, v2 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2"
    src.mkdir()
    vm.datagen_files(src, 77, 6, 256 * MiB)
    v1.mkdir(), v2.mkdir()
    vm.snapshot_tree(src, v1, None, None, shm_tmp / "v1.vmig")
    _flip(src / "f00002.bin", 3)
    (src / "f00005.bin").rename(src / "renamed.bin")
    vm.snapshot_tree(src, v2, v1, shm_tmp / "v1.vmig", shm_tmp / "v2.vmig")
    pairs = [(v1, shm_tmp / "v1.vmig"), (v2, shm_tmp / "v2.vmig")]
    report = shm_tmp / "scrub.txt"
    want = vm.scrub_store(pairs, report)                     # also warms the pipes: the thread / fd baseline
    report.unlink()
    threads, fds = _threads(), _fds()
    with vm.Ctl() as c:
        k = Canceller(c, lambda p: p["bytes_total"] and p["bytes_hashed"] >= 0.5 * p["bytes_total"])
        k.start()
        try:
            vm.scrub_store(pairs, report, ctl=c)
            res = None
        except vm.VmigError as e:
            res = e
        k.done.set()
        k.join()
        assert k.fired and res is not None and res.code == vm.VMIG_ECANCELED, res
        assert c.progress()["phase_name"] == "DATA"
    assert not report.exists() and not [n for n in os.listdir(shm_tmp) if n.startswith("scrub.txt")]
    again = vm.scrub_store(pairs, report)
    assert again["verdicts"] == want["verdicts"] == [vm.VMIG_OK] * 2 and again["bytes_unique"] == want["bytes_unique"]
    assert _threads() == threads and _fds() == fds


# ------------------------------------------------------------------------------------------ 7. hand-off
def test_scrub_replicaset_names_every_version(vm, orc, shm_tmp):
    import importlib
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ups = {f"rs-{i}": shm_tmp / f"upper_{i}" for i in (1, 2, 3)}
    _source(orc, ups["rs-1"])
    vm.set_resolver(container_upperdir=lambda n: str(ups[n]))
    ho.set_merges_root(shm_tmp)
    try:
        ho.SnapshotVersionIncremental("rs-1")
        ups["rs-2"].mkdir()
        orc.ref_copy(ups["rs-1"], ups["rs-2"])
        _flip(ups["rs-2"] / "data" / "g2.bin", 2 * BB)
        ho.SnapshotVersionIncremental("rs-2")
        ups["rs-3"].mkdir()
        orc.ref_copy(ups["rs-2"], ups["rs-3"])
        os.rename(ups["rs-3"] / "data" / "g1.bin", ups["rs-3"] / "g1_moved.bin")
        ho.SnapshotVersionIncremental("rs-3")
        (ho.versionDir("rs-4") / "diff").mkdir(parents=True)          # a snapshot that failed before its table
        (ho.versionDir("rs-x") / "diff").mkdir(parents=True)          # not a version
        out = ho.ScrubReplicaSet("rs")
        assert out["verdicts"] == {"rs-1": vm.VMIG_OK, "rs-2": vm.VMIG_OK, "rs-3": vm.VMIG_OK, "rs-4": vm.VMIG_ETABLE}
        assert out["report"] == shm_tmp / "merges" / "rs" / "scrub.txt"
        assert out["report"].read_bytes() == b"3\ttable\t.\t-\t-\t-\n"
        _flip(ho.snapshotPaths("rs-2")[0] / "data" / "g2.bin", 2 * BB + 1)    # the block rs-2 changed: not shared
        out = ho.ScrubReplicaSet("rs")
        assert out["verdicts"]["rs-2"] == vm.VMIG_ECORRUPT and out["verdicts"]["rs-1"] == vm.VMIG_OK
    finally:
        vm.set_resolver(None, None)
        ho.set_merges_root(None)
