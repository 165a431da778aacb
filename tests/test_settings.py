"""One workload under every option and environment setting an operator may turn (-m gpu), held to the oracle each time.

DESIGN.md §8: the host settings were chosen on one host type and every one of them is overridable.  An override may move
threads, slots, pipes, rings and NUMA placement, never a result.  So one workload -- a plain copy, a diff pass, a no-op
pass, an incremental snapshot, a checked restore of the whole snapshot and of one directory, and pageable and pinned
buffers -- runs unchanged under each setting at 64 KiB and 4 MiB blocks and must (a) pass every oracle check (the literal
tar pipe, block_table_of_tree, DESIGN.md §6's diff rule, C XXH64) and (b) give the digest of its deterministic outputs
that the default settings give.  Settings read once per process run in a child process of their own.  Where a setting
has an effect one can see, it is checked exactly: the reader, writer and slot counts of each lane from the VMIG_TRACE=1
line, lanes_used, files_direct, and the kernel launches of a one-lane plain copy (the packing rule of run_lane).

VMIG_F_MTIME_NS and VMIG_F_NO_METADATA, which change results on purpose, are pinned on their own below.
test_settings_host.py fails when a VMIG_F_* flag or a VMIG_* variable the engine reads is neither exercised here nor
on EXEMPT."""
import contextlib
import hashlib
import json
import os
import re
import stat
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

import _layer_model as L
from conftest import make_rich_tree

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BBS = (65536, 4 * MiB)
T0 = 1_600_000_000 * 10**9
HUGE = 4098 * 4096 + 333          # a block past 4095 at 4 KiB: where run_lane's 4096-block batch cap cuts
CHILD_TIMEOUT = 300               # seconds; a child that has not finished by then fails its test (never retried)
TOPS = ["A", "B", "Z", "_u", "a", "b", "z", "9", "10", "ü"]    # bytewise order differs from any locale's
STAT_KEYS = ("bytes_total", "bytes_written", "blocks_skipped", "blocks_total", "files_untrusted", "files", "dirs",
             "symlinks", "hardlinks", "specials")
SNAP_KEYS = ("files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled", "files_base_untrusted")

# Names the workload does not turn, each with the reason (test_settings_host.py reads this dict).
EXEMPT = {
    "VMIG_F_MOVE_SRC": "a move, not a copy option: test_gpu.py::test_move_matches_reference_mv against the literal mv",
    "VMIG_F_SKIP_HIDDEN_TOPDIRS": "the mv quirk a move needs: pinned with moves in test_gpu.py",
    "VMIG_F_PRUNE": "changes the result on purpose: the hand-off tests and test_versions.py hold it to the oracle",
    "VMIG_F_CUFILE": "needs the nvidia-fs driver: test_gpu.py's cufile variants skip without it",
    "VMIG_CUFILE": "the environment form of VMIG_F_CUFILE: needs the nvidia-fs driver",
    "VMIG_FAIL_BLOCK": "fault hook, tested in test_gpu.py",
    "VMIG_CORRUPT_BLOCK": "fault hook for VMIG_F_VERIFY, tested in test_gpu.py",
    "VMIG_PLAN_CPUS": "CPU-plan hook: test_host.py and test_concurrency.py",
    "VMIG_K1_PROXY_FENCE": "a K1 build variant: test_geometry.py runs it in a child process",
}


# ------------------------------------------------------------------------------------------ helpers
def _slot_bytes() -> int:
    return min(max(int(os.environ.get("VMIG_SLOT_MB", "32")), 4), 1024) << 20


def _slots() -> int:
    return min(max(int(os.environ.get("VMIG_SLOTS", "16")), 2), 64)


def io_rule(n: int):
    """vmig_opts.io_threads = n: (readers, writers) of every lane (include/vmig.h)."""
    if n == 1:
        return 1, 1
    r = (n + 1) * 2 // 5
    return r, n - r


def expected_launches(entries, second: set, bb: int, slot: int, align: int) -> int:
    """K1 launches of a one-lane plain copy, restated from run_lane: the planner lists the blocks of the written files
    (tree order, hard-link group once, empty files none) round-robin over groups of 64 files; consecutive blocks go into
    one batch while each takes align_up(max(len, 1), align) bytes of the slot and a batch has at most 4096 blocks."""
    sizes = [size for rel, size, _ in entries if rel not in second and size > 0]
    order = []
    for g in range(0, len(sizes), 64):
        grp = sizes[g:g + 64]
        for r in range(max(-(-s // bb) for s in grp)):
            order += [min(bb, s - r * bb) for s in grp if r * bb < s]
    batches, used, n = 0, 0, 0
    for ln in order:
        need = -(-max(ln, 1) // align) * align
        if n == 4096 or used + need > slot:
            batches, used, n = batches + 1, 0, 0
        used, n = used + need, n + 1
    return batches + (n > 0)


TRACE_RE = re.compile(r"reader busy \S+% of (\d+), writer busy \S+% of (\d+); dispatcher waited \S+ ms for (\d+) slots")


@contextlib.contextmanager
def _stderr_into(lines: list):
    """fd 2 into a temporary file while the block runs; its lines are appended to `lines`."""
    sys.stderr.flush()
    with tempfile.TemporaryFile() as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            yield
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            f.seek(0)
            lines.extend(f.read().decode(errors="replace").splitlines())


def _flip_first8(path, blocks, bb):
    with open(path, "r+b") as f:
        for b in blocks:
            f.seek(b * bb)
            w = bytes(x ^ 0xFF for x in f.read(8))
            f.seek(b * bb)
            f.write(w)


def _pin_times(root: Path) -> None:
    """Every entry gets an mtime fixed by its place in the tree; one in three falls on a whole second."""
    rels = sorted(os.path.relpath(os.path.join(d, n), root) for d, ds, fs in os.walk(root) for n in ds + fs)
    for k, rel in enumerate(reversed(rels + ["."])):
        t = T0 + k * 1_000_000_007 - (k * 1_000_000_007) % 10**9 * (k % 3 == 0)
        os.utime(root / rel, ns=(t, t), follow_symlinks=False)


def build_source(root: Path, orc) -> None:
    """The rich tree plus more than 8 top-level directories of many small files, one file of more than 4096 4 KiB blocks
    and a hard-link group that spans two top-level directories."""
    make_rich_tree(root / "rich", orc, seed=0x5E7, big=MiB + 777)
    for i, t in enumerate(TOPS):
        (root / t / "in").mkdir(parents=True)
        for j in range(12):
            (root / t / f"f{j:02d}").write_bytes(orc.splitmix_bytes(0x1000 + 100 * i + j, 1000 + 997 * j + 131 * i).tobytes())
        (root / t / "in" / "x").write_bytes(orc.splitmix_bytes(0x2000 + i, 70000 + i).tobytes())
    (root / "A" / "huge.bin").write_bytes(orc.splitmix_bytes(0xB16, HUGE).tobytes())
    os.link(root / "A" / "f00", root / "z" / "hl")
    _pin_times(root)


def flipped_blocks(bb: int) -> list:
    nb = -(-HUGE // bb)
    return sorted({0, 2, 3, 4, nb - 1, 4097 * 4096 // bb})


def _table_is(orc, path, bb, want) -> dict:
    """The engine's table at `path` equals the oracle's (entries, hashes) `want`; returns its digest part."""
    t = orc.read_table(path)
    entries, hashes = want
    assert t["block_bytes"] == bb and t["entries"] == entries, path
    bad = np.nonzero(t["hashes"] != hashes)[0]
    assert bad.size == 0, (str(path), bad[:10].tolist())
    return {"entries": [(os.fsdecode(r), s, f) for r, s, f in entries], "hashes": hashlib.sha256(hashes.tobytes()).hexdigest()}


def _same(want: dict, got: dict, what: str) -> None:
    d = L.diff_manifests(want, got)
    assert d == [], (what, d[:8])


class Source:
    """v1, v2 (v1 with blocks of A/huge.bin flipped), the tar pipe's copies of both and the oracle's tables, built once
    per process, block size and filesystem."""
    _cache = {}

    @classmethod
    def get(cls, orc, base: Path, bb: int) -> "Source":
        key = (str(base), bb)
        if key not in cls._cache:
            cls._cache[key] = cls(orc, base / f"src_{bb}", bb)
        return cls._cache[key]

    def __init__(self, orc, d: Path, bb: int):
        d.mkdir(parents=True)
        self.v1, self.v2 = d / "v1", d / "v2"
        self.v1.mkdir()
        build_source(self.v1, orc)
        L.freeze(self.v1, self.v2)
        huge = self.v2 / "A" / "huge.bin"
        t = os.lstat(huge).st_mtime_ns
        _flip_first8(huge, flipped_blocks(bb), bb)
        os.utime(huge, ns=(t, t))
        self.ref1, self.ref2 = d / "ref1", d / "ref2"
        for s, r in ((self.v1, self.ref1), (self.v2, self.ref2)):
            r.mkdir()
            orc.ref_copy(s, r)
        self.man1, self.man2 = orc.tree_manifest(self.ref1, mtime_ns=True), orc.tree_manifest(self.ref2, mtime_ns=True)
        self.tab1, self.tab2 = orc.block_table_of_tree(self.v1, bb), orc.block_table_of_tree(self.v2, bb)
        self.second = L.secondaries(orc.tree_manifest(self.v2))
        self.second_blocks = sum(-(-size // bb) for rel, size, _ in self.tab2[0] if rel in self.second)
        self.diff_want = L.expected_written(self.tab1, self.tab2, self.second, L.single_files(orc.tree_manifest(self.v1)), bb)
        self.noop_want = L.expected_written(self.tab2, self.tab2, self.second, L.single_files(orc.tree_manifest(self.v2)), bb)
        self.ring_want = L.expected_ring_bytes(self.tab1, self.tab2, self.second, bb)
        # a snapshot links every unchanged single-link file to the base's
        h1 = {rel: self.tab1[1][f:f + -(-s // bb)].tolist() for rel, s, f in self.tab1[0]}
        single = L.single_files(orc.tree_manifest(self.v2))
        self.linkable = sorted(os.fsdecode(rel) for rel, s, f in self.tab2[0]
                               if s and rel in single and h1.get(rel) == self.tab2[1][f:f + -(-s // bb)].tolist())
        assert self.diff_want[0] > 0 and self.linkable


# ------------------------------------------------------------------------------------------ the workload
def workload(vm, orc, base: Path, bb: int, run: str, opts: dict = None, flags: int = 0) -> dict:
    """Every step checked against the oracle.  Returns {"digest": the deterministic outputs' hash, "calls": per call its
    kind, the stats and the (readers, writers, slots) of every lane's VMIG_TRACE line}.  opts: io_threads,
    streams_per_gpu, lanes_per_gpu for every call; flags: added to every tree call."""
    o = dict(gpu_mask=1, block_bytes=bb, **(opts or {}))
    src = Source.get(orc, base, bb)
    w = base / f"{run}_{bb}"
    w.mkdir()
    calls, dig = [], {}

    def call(kind, fn, *a, **kw):
        lines = []
        with _stderr_into(lines):
            res = fn(*a, **kw)
        st = res[1] if isinstance(res, tuple) else res
        trace = [tuple(int(x) for x in m.groups()) for m in map(TRACE_RE.search, lines) if m]
        assert trace, (kind, lines[-5:])
        calls.append({"kind": kind, "stats": {k: v for k, v in st.items() if isinstance(v, int)}, "trace": trace})
        dig[kind] = {k: st[k] for k in STAT_KEYS + SNAP_KEYS if k in st}
        return res

    # plain copy into an empty directory
    dst = w / "dst"
    dst.mkdir()
    call("copy", vm.migrate_tree, src.v1, dst, None, w / "t1.vmig", flags=flags, **o)
    man = orc.tree_manifest(dst, mtime_ns=True)
    _same(src.man1, man, "copy")
    dig["copy_tree"], dig["copy_table"] = man, _table_is(orc, w / "t1.vmig", bb, src.tab1)
    # diff pass: known blocks flipped, against the destination's own table
    st = call("diff", vm.migrate_tree, src.v2, dst, w / "t1.vmig", w / "t2.vmig", flags=flags, **o)
    assert (st["blocks_total"] - st["blocks_skipped"] - src.second_blocks, st["bytes_written"]) == src.diff_want, st
    assert st["files_untrusted"] == 0, st
    man = orc.tree_manifest(dst, mtime_ns=True)
    _same(src.man2, man, "diff")
    dig["diff_tree"], dig["diff_table"] = man, _table_is(orc, w / "t2.vmig", bb, src.tab2)
    # no-op pass: only hard-link groups are written (never patched in place, DESIGN.md §6) and empty files made anew;
    # every other file keeps its inode and ctime
    ident = {p: (s.st_ino, s.st_ctime_ns) for p, s in ((p, os.lstat(p)) for p in dst.rglob("*")) if stat.S_ISREG(s.st_mode)
             and s.st_nlink == 1 and s.st_size}
    st = call("noop", vm.migrate_tree, src.v2, dst, w / "t2.vmig", w / "t3.vmig", flags=flags, **o)
    assert (st["blocks_total"] - st["blocks_skipped"] - src.second_blocks, st["bytes_written"]) == src.noop_want, st
    moved = [str(p) for p, v in ident.items() if (os.lstat(p).st_ino, os.lstat(p).st_ctime_ns) != v]
    assert moved == [], moved[:5]
    _same(src.man2, orc.tree_manifest(dst, mtime_ns=True), "noop")
    # incremental snapshot, then a checked restore of all of it and of one directory
    s1, s2 = w / "s1", w / "s2"
    s1.mkdir(), s2.mkdir()
    call("snap_base", vm.snapshot_tree, src.v1, s1, None, None, w / "s1.vmig", flags=flags, **o)
    st = call("snap_inc", vm.snapshot_tree, src.v2, s2, s1, w / "s1.vmig", w / "s2.vmig", flags=flags, **o)
    assert st["bytes_written"] == src.ring_want, st
    assert st["files_linked"] == len(src.linkable), (st, src.linkable)
    unlinked = [p for p in src.linkable if os.lstat(s2 / p).st_ino != os.lstat(s1 / p).st_ino]
    assert unlinked == [], unlinked
    _same(L.tree_in_itself(orc, src.ref2), L.tree_in_itself(orc, s2), "snapshot")
    dig["snap_table"] = _table_is(orc, w / "s2.vmig", bb, src.tab2)
    call("check", vm.restore_tree, s2, w / "s2.vmig", None, flags=vm.F_HASH_ONLY, **o)
    r1, r2 = w / "r1", w / "r2"
    r1.mkdir(), r2.mkdir()
    call("restore", vm.restore_tree, s2, w / "s2.vmig", r1, flags=flags | vm.F_VERIFY, **o)
    man = orc.tree_manifest(r1, mtime_ns=True)
    _same(src.man2, man, "restore_tree")
    call("paths", vm.restore_paths, s2, w / "s2.vmig", r2, ["B"], flags=flags | vm.F_VERIFY, **o)
    man = orc.tree_manifest(r2, mtime_ns=True)
    man.pop(".")
    _same({p: r for p, r in src.man2.items() if p == "B" or p.startswith("B/")}, man, "restore_paths")
    dig["paths_tree"] = man
    # host buffers with a prior: only the changed blocks are written
    n = 5 * MiB + 12345
    nb = -(-n // bb)
    offs = np.arange(nb, dtype=np.uint64) * bb
    lens = np.array([min(bb, n - b * bb) for b in range(nb)], np.uint32)
    data = orc.splitmix_bytes(0xB0F, n)
    prior = orc.hash_blocks(data, offs, lens)
    chosen = sorted({0, 1, nb - 1})
    new = data.copy()
    new[offs[chosen].astype(np.int64)] ^= 0xFF
    want = orc.hash_blocks(new, offs, lens)
    for kind in ("buffer_pageable", "buffer_pinned"):
        bufs = (vm.PinnedBuffer(n), vm.PinnedBuffer(n)) if kind == "buffer_pinned" else ()
        try:
            s, d = (bufs[0].array, bufs[1].array) if bufs else (np.empty(n, np.uint8), np.empty(n, np.uint8))
            s[:], d[:] = new, 0xEE
            h, st = call(kind, vm.migrate_buffer, s, d, prior, np.ones(nb, np.uint8), **o)
            assert (h == want).all(), np.nonzero(h != want)[0][:10]
            for b in range(nb):
                blk = slice(b * bb, b * bb + int(lens[b]))
                assert (d[blk] == new[blk]).all() if b in chosen else (d[blk] == 0xEE).all(), (kind, b)
            assert st["blocks_skipped"] == nb - len(chosen), st
            assert st["bytes_written"] == int(lens[chosen].astype(np.uint64).sum()), st
            dig[kind + "_hashes"] = [int(x) for x in h]
        finally:
            for x in bufs:
                x.free()
    # kernel launches of a one-lane plain copy follow run_lane's packing rule
    cp = calls[0]["stats"]
    direct = bool(flags & vm.F_DIRECT_IO) or os.environ.get("VMIG_DIRECT_IO") == "1"
    if cp["lanes_used"] == 1:
        want_k = expected_launches(src.tab1[0], L.secondaries(orc.tree_manifest(src.v1)), bb, _slot_bytes(), 4096 if direct else 512)
        assert cp["kernel_launches"] == want_k, (cp["kernel_launches"], want_k)
    return {"digest": hashlib.sha256(json.dumps(dig, sort_keys=True, default=list).encode()).hexdigest(), "calls": calls}


def _plan_checks(vm, calls) -> int:
    """Without io_threads, a one-lane diff pass and a hash-only check run the threads vmig_thread_plan says.  Returns
    how many calls it checked."""
    n = 0
    for c in calls:
        kinds = {"diff": dict(has_prior=True), "noop": dict(has_prior=True), "check": dict(flags=vm.F_HASH_ONLY)}
        if c["kind"] in kinds and c["stats"]["lanes_used"] == 1:
            want = vm.thread_plan(1, 1, **kinds[c["kind"]])
            assert [t[:2] for t in c["trace"]] == [want], (c["kind"], c["trace"], want)
            n += 1
    return n


def run_both(vm, orc, base: Path, run: str, **kw) -> dict:
    out = {"digest": {}, "calls": {}}
    for bb in BBS:
        r = workload(vm, orc, base, bb, run, **kw)
        out["digest"][str(bb)], out["calls"][str(bb)] = r["digest"], r["calls"]
    return out


# ------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def gpu(vm):
    vm.init(0)
    yield vm
    vm.shutdown()


@pytest.fixture(scope="module")
def work_dir():
    d = Path(tempfile.mkdtemp(prefix="vmig_set_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    yield d
    import shutil
    shutil.rmtree(d, ignore_errors=True)
    Source._cache.clear()


@pytest.fixture()
def traced(monkeypatch):
    monkeypatch.setenv("VMIG_TRACE", "1")      # read per lane run


@pytest.fixture(scope="module")
def default_run(gpu, orc, work_dir):
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("VMIG_TRACE", "1")
        return run_both(gpu, orc, work_dir, "default")


def test_default_settings(gpu, default_run):
    """The reference point of every other test here: the workload passes under the defaults, and its diff passes and
    hash-only check run the copy threads vmig_thread_plan reports."""
    for bb in BBS:
        assert _plan_checks(gpu, default_run["calls"][str(bb)]) == 3


# ------------------------------------------------------------------------------------------ ABI options, in process
@pytest.mark.parametrize("lanes", [1, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 64])
def test_io_threads_per_lane(gpu, orc, work_dir, default_run, traced, n, lanes):
    """vmig_opts.io_threads = n gives every lane exactly io_rule(n) readers and writers, whatever the call and however
    many lanes it has (n = 1: one of each, not the per-box budget)."""
    out = run_both(gpu, orc, work_dir, f"io{n}_l{lanes}", opts=dict(io_threads=n, lanes_per_gpu=lanes))
    assert out["digest"] == default_run["digest"]
    for bb in BBS:
        for c in out["calls"][str(bb)]:
            assert {t[:2] for t in c["trace"]} == {io_rule(n)}, (bb, c["kind"], c["trace"])
            if c["kind"] == "copy":
                assert c["stats"]["lanes_used"] == lanes and len(c["trace"]) == lanes, c


@pytest.mark.parametrize("lanes", [1, 3])
@pytest.mark.parametrize("s", [1, 2, 16, 17])
def test_streams_per_lane(gpu, orc, work_dir, default_run, traced, s, lanes):
    """vmig_opts.streams_per_gpu = s keeps min(s, the pipe's slots) slots in flight in every lane (17 > 16: all)."""
    out = run_both(gpu, orc, work_dir, f"st{s}_l{lanes}", opts=dict(streams_per_gpu=s, lanes_per_gpu=lanes))
    assert out["digest"] == default_run["digest"]
    for bb in BBS:
        for c in out["calls"][str(bb)]:
            assert {t[2] for t in c["trace"]} == {min(s, _slots())}, (bb, c["kind"], c["trace"])


# ------------------------------------------------------------------------------------------ environment, one child each
def _child_workload(a):
    """The engine half of test_environment_setting: the workload at both block sizes in this process's settings."""
    import __graft_entry__ as g
    from oracle import oracle as orc
    vm = g.load_pkg()
    vm.init(0)
    try:
        out = run_both(vm, orc, Path(a["base"]), "child", flags=a["flags"])
        out["plan_checked"] = sum(_plan_checks(vm, c) for c in out["calls"].values()) if a["plan"] else None
        if a["lanes2"]:
            (Path(a["base"]) / "l2").mkdir()
            out["lanes2"] = vm.migrate_tree(Source.get(orc, Path(a["base"]), BBS[0]).v1, Path(a["base"]) / "l2",
                                            gpu_mask=1, lanes_per_gpu=2)["lanes_used"]
        return out
    finally:
        vm.shutdown()


def _run_child(fn: str, arg: dict, env: dict) -> dict:
    here = Path(__file__).resolve().parent
    code = ("import json, sys; sys.path[:0] = sys.argv[1:3]; import test_settings as t; "
            "print(json.dumps(getattr(t, sys.argv[3])(json.loads(sys.argv[4]))))")
    r = subprocess.run([sys.executable, "-c", code, str(here), str(here.parent), fn, json.dumps(arg)],
                       env={**os.environ, "VMIG_TRACE": "1", **env}, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-6000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _fs_type(path) -> str:
    return subprocess.run(["stat", "-f", "-c", "%T", str(path)], capture_output=True, text=True).stdout.strip()


# (id, environment, on disk, flags of every tree call)
ENV_ROWS = [
    ("readers1", {"VMIG_READERS": "1", "VMIG_WRITERS": "1"}, False, 0),
    ("readers64", {"VMIG_READERS": "64", "VMIG_WRITERS": "64"}, False, 0),
    ("io_share8", {"VMIG_IO_SHARE": "8"}, False, 0),
    ("huge0", {"VMIG_HUGE": "0"}, False, 0),
    ("huge0_direct_disk", {"VMIG_HUGE": "0"}, True, "F_DIRECT_IO"),
    ("numa0", {"VMIG_NUMA": "0"}, False, 0),
    ("bind_io0", {"VMIG_BIND_IO": "0"}, False, 0),
    ("bind_writers1", {"VMIG_BIND_WRITERS": "1"}, False, 0),
    ("rings_far_near", {"VMIG_RING_IN_NODE": "1", "VMIG_RING_OUT_NODE": "0"}, False, 0),
    ("rings_alternate", {"VMIG_RING_IN_NODE": "2", "VMIG_RING_OUT_NODE": "2"}, False, 0),
    ("ring_mbind", {"VMIG_RING_MBIND": "1"}, False, 0),
    ("walk1", {"VMIG_WALK_THREADS": "1"}, False, 0),
    ("walk32", {"VMIG_WALK_THREADS": "32"}, False, 0),
    ("lanes3", {"VMIG_LANES_PER_GPU": "3"}, False, 0),
    ("direct_env_tmpfs", {"VMIG_DIRECT_IO": "1"}, False, 0),
    ("direct_env_disk", {"VMIG_DIRECT_IO": "1"}, True, 0),
    ("slot64x2", {"VMIG_SLOT_MB": "64", "VMIG_SLOTS": "2"}, False, 0),
    ("slot4x64", {"VMIG_SLOT_MB": "4", "VMIG_SLOTS": "64"}, False, 0),
    ("pipes8", {"VMIG_PIPES_PER_GPU": "8"}, False, 0),
]


@pytest.mark.parametrize("env,disk,flags", [r[1:] for r in ENV_ROWS], ids=[r[0] for r in ENV_ROWS])
def test_environment_setting(gpu, orc, work_dir, default_run, tmp_path, env, disk, flags):
    """Each environment knob in a process of its own (the engine reads most of them once per process): the workload's
    oracle checks pass there, its digest is the default one, and the knob's visible effect is exact."""
    base = tmp_path if disk else work_dir / ("env_" + "_".join(f"{k}{v}" for k, v in sorted(env.items())))
    base.mkdir(exist_ok=True)
    flag_bits = getattr(gpu, flags) if flags else 0
    io_default = not ({"VMIG_READERS", "VMIG_LANES_PER_GPU"} & set(env))
    out = _run_child("_child_workload", {"base": str(base), "flags": flag_bits, "plan": io_default,
                                         "lanes2": "VMIG_LANES_PER_GPU" in env}, env)
    assert out["digest"] == default_run["digest"]
    calls = [dict(c, trace=[tuple(t) for t in c["trace"]]) for bb in BBS for c in out["calls"][str(bb)]]
    traces = {t for c in calls for t in c["trace"]}
    if "VMIG_READERS" in env:
        assert {t[:2] for t in traces} == {(int(env["VMIG_READERS"]), int(env["VMIG_WRITERS"]))}, traces
    if io_default:
        assert out["plan_checked"] == 6, out["plan_checked"]
    if "VMIG_IO_SHARE" in env:          # the plan the child followed is not the one this process (share 1) makes
        diff = next(c for c in calls if c["kind"] == "diff")
        assert diff["trace"][0][:2] != gpu.thread_plan(1, 1, has_prior=True), diff["trace"]
    if "VMIG_SLOTS" in env:
        assert {t[2] for t in traces} == {int(env["VMIG_SLOTS"])}, traces
    if "VMIG_LANES_PER_GPU" in env:
        assert all(c["stats"]["lanes_used"] == 3 for c in calls if c["kind"] in ("copy", "diff", "snap_base")), calls
        assert out["lanes2"] == 2
    if disk and _fs_type(tmp_path) not in ("tmpfs", "ramfs"):
        assert all(c["stats"]["files_direct"] > 0 for c in calls if c["kind"] in ("copy", "snap_base", "restore")), calls


# ------------------------------------------------------------------------------------------ VMIG_F_MTIME_NS
def _ns_tree(root: Path, orc) -> list:
    """Files without hard links, half of them with nanoseconds in their mtime; returns those paths."""
    (root / "d").mkdir(parents=True)
    for i in range(8):
        (root / ("d" if i % 2 else ".") / f"m{i}").write_bytes(orc.splitmix_bytes(0x700 + i, 3000 + 70001 * i).tobytes())
    ns = []
    for i, p in enumerate(sorted(root.rglob("m*"))):
        t = T0 + i * 10**9 + (123456789 if i % 2 == 0 else 0)
        os.utime(p, ns=(t, t))
        if t % 10**9:
            ns.append(os.path.relpath(p, root))
    os.utime(root / "d", ns=(T0 + 7, T0 + 7))
    os.utime(root, ns=(T0 + 9, T0 + 9))
    return ns


def _ids(root: Path, rels) -> dict:
    return {r: (os.lstat(root / r).st_ino, os.lstat(root / r).st_ctime_ns) for r in rels}


def test_mtime_ns_copy_keeps_every_mtime(gpu, orc, shm_tmp):
    """With VMIG_F_MTIME_NS every entry -- files, directories and the root, symlinks, specials -- keeps its mtime to the
    nanosecond; everything else is what the tar pipe gives.  Without it the copy is the tar pipe's at whole seconds."""
    src, dst, plain, ref = (shm_tmp / n for n in ("src", "dst", "plain", "ref"))
    for d in (src, dst, plain, ref):
        d.mkdir()
    build_source(src, orc)
    orc.ref_copy(src, ref)
    gpu.migrate_tree(src, dst, flags=gpu.F_MTIME_NS, gpu_mask=1)
    want, src_ns = orc.tree_manifest(ref, mtime_ns=True), orc.tree_manifest(src, mtime_ns=True)
    assert any(r["mtime"] % 10**9 for r in src_ns.values())
    for rel, r in want.items():
        r["mtime"] = src_ns[rel]["mtime"]
    _same(want, orc.tree_manifest(dst, mtime_ns=True), "mtime_ns copy")
    gpu.migrate_tree(src, plain, gpu_mask=1)
    assert orc.compare_trees(ref, plain, mtime_ns=True) == []


@pytest.mark.parametrize("first", [True, False], ids=["ns-then-seconds", "seconds-then-ns"])
def test_mtime_ns_switched_between_passes(gpu, orc, shm_tmp, first):
    """A table written with one VMIG_F_MTIME_NS setting, then two passes with the other over an unchanged source: the
    first of them writes no data but puts each file's mtime as its flag says, which moves the ctimes of exactly the files
    whose mtime has nanoseconds, and records them; the second touches nothing."""
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    dst.mkdir()
    src.mkdir()
    ns = _ns_tree(src, orc)
    files = sorted(os.path.relpath(p, src) for p in src.rglob("m*"))
    f1 = gpu.F_MTIME_NS if first else 0
    f2 = 0 if first else gpu.F_MTIME_NS
    gpu.migrate_tree(src, dst, None, shm_tmp / "t1", flags=f1, gpu_mask=1)
    before = _ids(dst, files)
    st = gpu.migrate_tree(src, dst, shm_tmp / "t1", shm_tmp / "t2", flags=f2, gpu_mask=1)
    assert st["bytes_written"] == 0 and st["files_untrusted"] == 0, st
    after = _ids(dst, files)
    assert sorted(r for r in files if after[r] != before[r]) == ns
    assert all(after[r][0] == before[r][0] for r in files)           # patched in place, never replaced
    for r in files:
        m = os.lstat(src / r).st_mtime_ns
        assert os.lstat(dst / r).st_mtime_ns == (m if f2 else m - m % 10**9), r
    t2 = orc.read_table(shm_tmp / "t2")
    assert dict(zip((os.fsdecode(e[0]) for e in t2["entries"]), t2["identity"])) == {r: tuple(after[r]) for r in files}
    st = gpu.migrate_tree(src, dst, shm_tmp / "t2", shm_tmp / "t3", flags=f2, gpu_mask=1)
    assert st["bytes_written"] == 0 and _ids(dst, files) == after, st


@pytest.mark.parametrize("f_base,f_inc", [(0, 0), (1, 1), (0, 1), (1, 0)], ids=["s-s", "ns-ns", "s-ns", "ns-s"])
def test_mtime_ns_snapshot_links(gpu, orc, shm_tmp, f_base, f_inc):
    """DESIGN.md §6: an increment links a base file only when the base inode already carries the mtime the copy would
    get under the increment's own flags.  The same flags: every file is linked.  Different flags: exactly the files
    whose mtime is a whole second.  Both snapshots restore to the tar pipe's copy."""
    src, ref, s1, s2 = (shm_tmp / n for n in ("src", "ref", "s1", "s2"))
    for d in (ref, s1, s2, src):
        d.mkdir()
    ns = _ns_tree(src, orc)
    orc.ref_copy(src, ref)
    files = sorted(os.path.relpath(p, src) for p in src.rglob("m*"))
    fl = lambda f: gpu.F_MTIME_NS if f else 0
    gpu.snapshot_tree(src, s1, None, None, shm_tmp / "s1.vmig", flags=fl(f_base), gpu_mask=1)
    st = gpu.snapshot_tree(src, s2, s1, shm_tmp / "s1.vmig", shm_tmp / "s2.vmig", flags=fl(f_inc), gpu_mask=1)
    linked = sorted(r for r in files if os.lstat(s2 / r).st_ino == os.lstat(s1 / r).st_ino)
    want = files if f_base == f_inc else sorted(set(files) - set(ns))
    assert linked == want and st["files_linked"] == len(want) and st["bytes_written"] == 0, st
    for i, (snap, tab) in enumerate(((s1, "s1.vmig"), (s2, "s2.vmig"))):
        r = shm_tmp / f"r{i}"
        r.mkdir()
        gpu.restore_tree(snap, shm_tmp / tab, r, gpu_mask=1, flags=gpu.F_VERIFY)
        assert orc.compare_trees(ref, r, mtime_ns=True) == [], snap


# ------------------------------------------------------------------------------------------ VMIG_F_NO_METADATA
def _meta(root: Path) -> dict:
    out = {}
    for p in [root] + sorted(root.rglob("*")):
        s = os.lstat(p)
        out[os.path.relpath(p, root)] = (stat.S_IMODE(s.st_mode), s.st_uid, s.st_gid, s.st_mtime_ns)
    return out


def _umask() -> int:
    um = os.umask(0o022)
    os.umask(um)
    return um


def test_no_metadata_copies_data_only(gpu, orc, shm_tmp):
    """VMIG_F_NO_METADATA: contents, kinds, symlink targets, hard-link groups and device numbers are the tar pipe's; what
    the call creates has the engine's creation modes less the umask (files and specials 0600, directories 0700) and the
    caller as owner; the root keeps its mode.  A diff pass then leaves owner, mode and mtime of the directories and of
    the files it patches alone (mtime: unless it writes into them) and still skips every unchanged block."""
    bb = 65536
    src = Source.get(orc, shm_tmp, bb)
    dst = shm_tmp / "dst"
    dst.mkdir(mode=0o751)
    os.chmod(dst, 0o751)
    gpu.migrate_tree(src.v1, dst, None, shm_tmp / "t1", flags=gpu.F_NO_METADATA, block_bytes=bb, gpu_mask=1)
    strip = lambda m: {p: {k: v for k, v in r.items() if k not in ("mode", "uid", "gid", "mtime")} for p, r in m.items()}
    got = orc.tree_manifest(dst, mtime_ns=True)
    _same(strip(src.man1), strip(got), "no_metadata copy")
    um = _umask()
    for rel, r in got.items():
        want = 0o751 if rel == "." else None if stat.S_ISLNK(r["type"]) else (0o700 if stat.S_ISDIR(r["type"]) else 0o600) & ~um
        if want is not None:
            assert r["mode"] == want, (rel, oct(r["mode"]), oct(want))
        if rel != ".":
            assert (r["uid"], r["gid"]) == (os.geteuid(), os.getegid()), rel
    # pre-existing directories with their own mode and mtime; the files stay as the copy left them (trusted)
    for d, mode in (("rich/sub/deep", 0o755), ("B/in", 0o705)):
        os.chmod(dst / d, mode)
        os.utime(dst / d, ns=(T0 + 5, T0 + 5))
    before = _meta(dst)
    st = gpu.migrate_tree(src.v2, dst, shm_tmp / "t1", shm_tmp / "t2", flags=gpu.F_NO_METADATA, block_bytes=bb, gpu_mask=1)
    assert (st["blocks_total"] - st["blocks_skipped"] - src.second_blocks, st["bytes_written"]) == src.diff_want, st
    assert st["files_untrusted"] == 0, st
    after = _meta(dst)
    single = {os.fsdecode(r) for r in L.single_files(orc.tree_manifest(src.v1))}
    for rel, (mode, uid, gid, mt) in before.items():
        kind = got.get(rel, {}).get("type")
        if kind == stat.S_IFDIR or rel in single:
            assert after[rel][:3] == (mode, uid, gid), (rel, before[rel], after[rel])
        if rel in single and got[rel]["size"] and rel != "A/huge.bin" or rel in ("rich/sub/deep", "B/in"):
            assert after[rel][3] == mt, (rel, before[rel], after[rel])
    assert (dst / "A" / "huge.bin").read_bytes() == (src.v2 / "A" / "huge.bin").read_bytes()


@pytest.mark.skipif(os.geteuid() == 0, reason="root opens a read-only file for writing without lending it a write bit")
def test_no_metadata_read_only_file_keeps_its_mode(gpu, orc, shm_tmp):
    """As an ordinary user, a read-only destination file the diff pass patches in place is lent a write bit; under
    VMIG_F_NO_METADATA it gets its own mode back, written to or not."""
    src, dst = shm_tmp / "src", shm_tmp / "dst"
    src.mkdir(), dst.mkdir()
    for n in ("chg.bin", "same.bin"):
        (src / n).write_bytes(orc.splitmix_bytes(len(n), 3 * 65536 + 5).tobytes())
        os.chmod(src / n, 0o444)
    gpu.migrate_tree(src, dst, None, shm_tmp / "t1", block_bytes=65536, gpu_mask=1)
    before = _meta(dst)
    assert before["chg.bin"][0] == 0o444 & ~_umask()
    os.chmod(src / "chg.bin", 0o644)
    _flip_first8(src / "chg.bin", [1], 65536)
    os.chmod(src / "chg.bin", 0o444)
    st = gpu.migrate_tree(src, dst, shm_tmp / "t1", None, flags=gpu.F_NO_METADATA, block_bytes=65536, gpu_mask=1)
    assert st["bytes_written"] == 65536 and st["files_untrusted"] == 0, st
    after = _meta(dst)
    assert {n: after[n][0] for n in ("chg.bin", "same.bin")} == {n: before[n][0] for n in ("chg.bin", "same.bin")}
    assert (dst / "chg.bin").read_bytes() == (src / "chg.bin").read_bytes()
