"""Calls of every kind at once on one GPU (-m gpu), each held to the oracle while they share the staging pipes.

include/vmig.h promises that every entry point is re-entrant and thread-safe.  All data-path calls check their staging
pipes out of one per-GPU pool, and each call hands its pipe (16 slots: stream, pinned rings, HBM buffer, descriptor and
result areas, events, K1 work counter) to whichever call comes next.  A job below is one call with its own directories,
its own control and its own expectation.  Every expectation comes from the oracle (C XXH64, the literal tar pipe,
block_table_of_tree), from numpy or from tests/_layer_model.py, and is computed before any thread starts.  The
deterministic counters of each call are also pinned to what the same job returns when it runs alone.

The jobs use different block sizes on purpose, so a slot last used at one geometry and in one mode (hash-only, diff,
plain copy, per-block DMA from a pinned buffer, restore with expected hashes) is reused at another.  One job fails
(VMIG_ECORRUPT) and one is cancelled: both must give their pipes back for the calls that wait."""
import json
import os
import re
import shutil
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import pytest

import _layer_model as L
from conftest import make_rich_tree
from test_gpu import ring_boundary_case

pytestmark = pytest.mark.gpu
MiB = 1 << 20
T0 = 1_500_000_000_000_000_000
JOIN_S = 300                       # a call of the mix that has not returned by then is stuck waiting for a pipe
# the counters a call computes from its inputs alone: the same whatever runs beside it
PINNED = ("bytes_total", "blocks_total", "blocks_skipped", "bytes_written", "bytes_h2d", "bytes_d2h", "files", "lanes_used",
          "kernel_launches")


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


# ------------------------------------------------------------------------------------------ helpers
def _flip_first8(path, blocks, bb):
    """Invert the first (up to) 8 bytes of each block in place."""
    with open(path, "r+b") as f:
        for b in blocks:
            f.seek(b * bb)
            w = bytes(x ^ 0xFF for x in f.read(8))
            f.seek(b * bb)
            f.write(w)


def _flip_byte(path, off):
    with open(path, "r+b") as f:
        f.seek(off)
        x = f.read(1)[0]
        f.seek(off)
        f.write(bytes([x ^ 0x5A]))


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


def _table_is(orc, path, bb, root):
    entries, want = orc.block_table_of_tree(root, bb)
    t = orc.read_table(path)
    assert t["block_bytes"] == bb and t["entries"] == entries, path
    bad = np.nonzero(t["hashes"] != want)[0]
    assert bad.size == 0, (str(path), bad[:10].tolist())


def _no_table_left(path: Path):
    assert not path.exists(), path
    assert not [n for n in os.listdir(path.parent) if n.startswith(path.name + ".tmp")], os.listdir(path.parent)


def _foreign(msg: str, own: str) -> set:
    """The tags of other jobs (their directory and file names start with jNN_) that an error text mentions."""
    return set(re.findall(r"j\d\d_", msg)) - {own[:4]}


def _blen(size, bb, b):
    return min(bb, size - b * bb)


class Outcome:
    def __init__(self, res, err, msg, progress):
        self.res, self.err, self.msg, self.progress = res, err, msg, progress

    def stats(self):
        """The call's vmig_stats (None for calls that have none)."""
        if isinstance(self.res, tuple) and isinstance(self.res[1], dict):     # migrate_buffer: (hashes, stats)
            return self.res[1]
        if isinstance(self.res, dict):
            return self.res.get("stats", self.res)  # scrub_store nests the data pass's counters
        return None


class Job:
    """One call: stage(run) prepares its per-run inputs serially, call(s, ctl) runs in a thread of the mix, check(s, out)
    holds the outcome to the oracle.  uses_ctl: the call gets its own Ctl."""
    name = "?"
    uses_ctl = False
    progress_is_stats = False       # a successful call's final progress must equal its stats (include/vmig.h)

    def __init__(self, vm, orc, base: Path):
        self.vm, self.orc, self.base = vm, orc, base / self.name
        self.base.mkdir()

    def stage(self, run: str) -> dict:
        d = self.base / run
        d.mkdir()
        return {"dir": d}

    def release(self, s: dict):
        shutil.rmtree(s["dir"], ignore_errors=True)


# 1. plain copy of the rich tree at 4 MiB, with an out table
class CopyJob(Job):
    name, uses_ctl, progress_is_stats = "j01_copy", True, True

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        self.src, self.ref = self.base / "src", self.base / "ref"
        self.src.mkdir(), self.ref.mkdir()
        make_rich_tree(self.src, orc, seed=101)
        orc.ref_copy(self.src, self.ref)

    def stage(self, run):
        s = super().stage(run)
        (s["dir"] / "dst").mkdir()
        return s

    def call(self, s, ctl):
        return self.vm.migrate_tree(self.src, s["dir"] / "dst", None, s["dir"] / "t.vmig", ctl=ctl)

    def check(self, s, out):
        assert self.orc.compare_trees(self.ref, s["dir"] / "dst", mtime_ns=True) == []
        _table_is(self.orc, s["dir"] / "t.vmig", 4 * MiB, self.src)


# 2. diff pass at 64 KiB against the destination's own table, chosen blocks changed; 10. the same with three lanes
class DiffJob(Job):
    name, uses_ctl, progress_is_stats = "j02_diff", True, True
    bb, lanes = 65536, 0

    def _sources(self, v1, v2):
        make_rich_tree(v1, self.orc, seed=102)
        (v1 / "j02_huge.bin").write_bytes(self.orc.splitmix_bytes(0x202, 7 * MiB + 4097).tobytes())
        L.freeze(v1, v2)
        nb = -(-(7 * MiB + 4097) // self.bb)
        _flip_first8(v2 / "j02_huge.bin", [0, 1, 40, 41, 42, nb - 1], self.bb)
        _flip_first8(v2 / "exact.bin", [3], self.bb)

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        v1, self.src, self.ref = self.base / "v1", self.base / "v2", self.base / "ref"
        v1.mkdir()
        self._sources(v1, self.src)
        self.ref.mkdir()
        orc.ref_copy(self.src, self.ref)
        self.v1 = v1
        tab1, tab2 = orc.block_table_of_tree(v1, self.bb), orc.block_table_of_tree(self.src, self.bb)
        second = L.secondaries(orc.tree_manifest(self.src))
        self.second_blocks = sum(-(-size // self.bb) for rel, size, _ in tab2[0] if rel in second)
        # the destination holds v1 as tar left it: its single-link files are patched in place
        self.want_written = L.expected_written(tab1, tab2, second, L.single_files(orc.tree_manifest(v1)), self.bb)
        assert self.want_written[0] > 0

    def stage(self, run):
        s = super().stage(run)
        dst = s["dir"] / "dst"
        dst.mkdir()
        self.orc.ref_copy(self.v1, dst)
        self.vm.hash_tree(dst, s["dir"] / "prior.vmig", block_bytes=self.bb)
        _table_is(self.orc, s["dir"] / "prior.vmig", self.bb, self.v1)
        return s

    def call(self, s, ctl):
        return self.vm.migrate_tree(self.src, s["dir"] / "dst", s["dir"] / "prior.vmig", s["dir"] / "t.vmig",
                                    block_bytes=self.bb, lanes_per_gpu=self.lanes, ctl=ctl)

    def check(self, s, out):
        st = out.res
        assert self.orc.compare_trees(self.ref, s["dir"] / "dst", mtime_ns=True) == []
        _table_is(self.orc, s["dir"] / "t.vmig", self.bb, self.src)
        got = (st["blocks_total"] - st["blocks_skipped"] - self.second_blocks, st["bytes_written"])
        assert got == self.want_written, (got, self.want_written, st)
        assert st["files_untrusted"] == 0, st
        if self.lanes:
            assert st["lanes_used"] == self.lanes, st


class DiffLanesJob(DiffJob):
    name = "j10_diff3"
    bb, lanes = MiB, 3

    def _sources(self, v1, v2):
        for i in range(8):
            (v1 / f"j10_f{i}.bin").write_bytes(self.orc.splitmix_bytes(0x1000 + i, (i + 2) * MiB + 333 * i).tobytes())
        (v1 / "sub").mkdir()
        (v1 / "sub" / "j10_small").write_bytes(b"s" * 5000)
        L.freeze(v1, v2)
        _flip_first8(v2 / "j10_f1.bin", [0, 2], self.bb)
        _flip_first8(v2 / "j10_f6.bin", [7], self.bb)
        os.truncate(v2 / "j10_f4.bin", 3 * MiB + 5)
        (v2 / "j10_new.bin").write_bytes(self.orc.splitmix_bytes(0x10FF, 2 * MiB + 1).tobytes())


# 3. incremental snapshot at 4 KiB against a base: a moved file and a changed file
class SnapshotJob(Job):
    name = "j03_snap"
    bb = 4096
    CHG = 2 * MiB + 100

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        self.v1, self.src, self.ref = self.base / "v1", self.base / "v2", self.base / "ref"
        (self.v1 / "old").mkdir(parents=True)
        (self.v1 / "j03_keep.bin").write_bytes(orc.splitmix_bytes(0x301, 300 * 1024 + 7).tobytes())
        (self.v1 / "old" / "j03_moved.bin").write_bytes(orc.splitmix_bytes(0x302, MiB + 5).tobytes())
        (self.v1 / "j03_chg.bin").write_bytes(orc.splitmix_bytes(0x303, self.CHG).tobytes())
        L.freeze(self.v1, self.src)
        (self.src / "new").mkdir()
        os.rename(self.src / "old" / "j03_moved.bin", self.src / "new" / "j03_moved.bin")
        nb = -(-self.CHG // self.bb)
        self.chosen = [0, 17, 200, 201, nb - 1]
        _flip_first8(self.src / "j03_chg.bin", self.chosen, self.bb)
        self.ref.mkdir()
        orc.ref_copy(self.src, self.ref)
        self.want_tree = L.tree_in_itself(orc, self.ref)

    def stage(self, run):
        s = super().stage(run)
        (s["dir"] / "base").mkdir(), (s["dir"] / "v2").mkdir()
        self.vm.snapshot_tree(self.v1, s["dir"] / "base", None, None, s["dir"] / "base.vmig", block_bytes=self.bb)
        _table_is(self.orc, s["dir"] / "base.vmig", self.bb, self.v1)
        return s

    def call(self, s, ctl):
        d = s["dir"]
        return self.vm.snapshot_tree(self.src, d / "v2", d / "base", d / "base.vmig", d / "v2.vmig", block_bytes=self.bb,
                                     ctl=ctl)

    def check(self, s, out):
        st = out.res
        assert L.diff_manifests(self.want_tree, L.tree_in_itself(self.orc, s["dir"] / "v2")) == []
        _table_is(self.orc, s["dir"] / "v2.vmig", self.bb, self.src)
        assert st["files_linked"] == 2 and st["files_backfilled"] == 1 and st["files_base_untrusted"] == 0, st
        assert st["bytes_backfilled"] == self.CHG - sum(_blen(self.CHG, self.bb, b) for b in self.chosen), st

    def same_as_alone(self, out, alone):
        keys = ("files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled", "files_base_untrusted")
        assert {k: out.res[k] for k in keys} == {k: alone.res[k] for k in keys}


# 4. restore of a snapshot with one byte flipped in a known block: VMIG_ECORRUPT naming that path and block
class RestoreCorruptJob(Job):
    name = "j04_rot"
    bb = 131072
    SIZE = 3 * MiB + 99
    OFF = 9 * 131072 + 77

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        src, self.snap, self.table = self.base / "src", self.base / "snap", self.base / "snap.vmig"
        src.mkdir(), self.snap.mkdir()
        (src / "j04_ok.bin").write_bytes(orc.splitmix_bytes(0x401, MiB + 3).tobytes())
        body = orc.splitmix_bytes(0x402, self.SIZE)
        (src / "j04_rot.bin").write_bytes(body.tobytes())
        vm.migrate_tree(src, self.snap, None, self.table, block_bytes=self.bb)
        _table_is(orc, self.table, self.bb, src)
        _flip_byte(self.snap / "j04_rot.bin", self.OFF)
        k = self.OFF // self.bb
        bad = body.copy()
        bad[self.OFF] ^= 0x5A
        got = orc.xxh64(bad[k * self.bb:(k + 1) * self.bb].tobytes())
        want = orc.xxh64(body[k * self.bb:(k + 1) * self.bb].tobytes())
        self.want_msg = f"j04_rot.bin block {k} hashes {got:016x}, its block table says {want:016x}"

    def stage(self, run):
        s = super().stage(run)
        (s["dir"] / "dst").mkdir()
        return s

    def call(self, s, ctl):
        return self.vm.restore_tree(self.snap, self.table, s["dir"] / "dst", None, s["dir"] / "t.vmig", block_bytes=self.bb,
                                    ctl=ctl)

    def check(self, s, out):
        assert out.err == self.vm.VMIG_ECORRUPT, (out.err, out.res)
        assert out.msg.endswith(self.want_msg), out.msg
        assert not _foreign(out.msg, self.name) and "cancel" not in out.msg, out.msg      # no other job's text
        _no_table_left(s["dir"] / "t.vmig")


# 5. scrub of a store of three versions, the last one damaged
class ScrubJob(Job):
    name = "j05_scrub"
    bb = 262144

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        src = self.base / "src"
        src.mkdir()
        a = orc.splitmix_bytes(0x501, MiB + 3)
        (src / "j05_a.bin").write_bytes(a.tobytes())
        (src / "j05_b.bin").write_bytes(orc.splitmix_bytes(0x502, 700 * 1024).tobytes())
        self.pairs = []
        for v in range(3):
            if v == 1:
                _flip_first8(src / "j05_b.bin", [1], self.bb)
            if v == 2:
                _flip_first8(src / "j05_a.bin", [0], self.bb)
                a = np.fromfile(src / "j05_a.bin", np.uint8)
            d, t = self.base / f"v{v}", self.base / f"v{v}.vmig"
            d.mkdir()
            prev = self.pairs[-1] if self.pairs else (None, None)
            vm.snapshot_tree(src, d, prev[0], prev[1], t, block_bytes=self.bb)
            _table_is(orc, t, self.bb, src)
            self.pairs.append((d, t))
        off = 2 * self.bb + 1000                  # v2's own copy of j05_a.bin (it changed in v2), block 2
        _flip_byte(self.pairs[2][0] / "j05_a.bin", off)
        bad = a.copy()
        bad[off] ^= 0x5A
        blk = slice(2 * self.bb, 3 * self.bb)
        self.want_findings = [{"version": 2, "kind": "block", "path": "j05_a.bin", "block": 2,
                               "got": orc.xxh64(bad[blk].tobytes()), "want": orc.xxh64(a[blk].tobytes())}]

    def call(self, s, ctl):
        return self.vm.scrub_store(self.pairs, s["dir"] / "report.txt", block_bytes=self.bb, ctl=ctl)

    def check(self, s, out):
        r = out.res
        vm = self.vm
        assert r["verdicts"] == [vm.VMIG_OK, vm.VMIG_OK, vm.VMIG_ECORRUPT], r["verdicts"]
        assert r["findings"] == self.want_findings, r["findings"]

    def same_as_alone(self, out, alone):
        a, b = dict(out.res), dict(alone.res)
        a.pop("stats"), b.pop("stats")
        assert a == b


# 6. restore of two chosen paths into a populated layer
class RestorePathsJob(Job):
    name = "j06_paths"
    bb = 12288
    PATHS = ["j06_p1.bin", "sub/j06_p2.bin"]

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        src, self.snap, self.table = self.base / "src", self.base / "snap", self.base / "snap.vmig"
        (src / "sub").mkdir(parents=True), self.snap.mkdir()
        (src / "j06_p1.bin").write_bytes(orc.splitmix_bytes(0x601, 200 * 1024 + 1).tobytes())
        (src / "sub" / "j06_p2.bin").write_bytes(orc.splitmix_bytes(0x602, MiB + 12287).tobytes())
        (src / "j06_other.bin").write_bytes(orc.splitmix_bytes(0x603, 50000).tobytes())
        (src / "sub" / "j06_q.bin").write_bytes(b"q" * 7)
        vm.migrate_tree(src, self.snap, None, self.table, block_bytes=self.bb)
        _table_is(orc, self.table, self.bb, src)
        man = orc.tree_manifest(self.snap, mtime_ns=True)
        self.want = {p: man[p] for p in self.PATHS}

    def stage(self, run):
        s = super().stage(run)
        dst = s["dir"] / "dst"
        (dst / "sub").mkdir(parents=True)
        (dst / "j06_p1.bin").write_bytes(b"old" * 1000)
        (dst / "j06_other.bin").write_bytes(b"not from the snapshot")
        (dst / "sub" / "j06_keep").write_bytes(b"k")
        (dst / "j06_stale").mkdir()
        for p in (dst / "j06_p1.bin", dst / "j06_other.bin", dst / "sub" / "j06_keep", dst / "j06_stale", dst / "sub", dst):
            os.utime(p, ns=(T0, T0))
        s["before"] = _state(dst)
        return s

    def call(self, s, ctl):
        return self.vm.restore_paths(self.snap, self.table, s["dir"] / "dst", self.PATHS, block_bytes=self.bb, ctl=ctl)

    def check(self, s, out):
        dst = s["dir"] / "dst"
        man = self.orc.tree_manifest(dst, mtime_ns=True)
        assert {p: man.get(p) for p in self.PATHS} == self.want
        after = _state(dst)
        for rel, v in s["before"].items():
            if rel not in (".", "sub") and rel not in self.PATHS:
                assert after.get(rel) == v, rel
        assert set(after) == set(s["before"]) | {"sub/j06_p2.bin"}, sorted(after)


# 7. K1 direct on the ring-boundary length set
class HashBlocksJob(Job):
    name = "j07_k1"

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        self.buf, self.offs, self.lens = ring_boundary_case()
        self.want = orc.hash_blocks(self.buf, self.offs, self.lens)

    def call(self, s, ctl):
        return self.vm.hash_blocks(self.buf, self.offs, self.lens)[0]

    def check(self, s, out):
        bad = np.nonzero(out.res != self.want)[0]
        assert bad.size == 0, [(int(i), int(self.lens[i])) for i in bad[:10]]


# 8. host buffer to host buffer at 64 KiB, prior hashes skip the unchanged blocks; pinned (per-block DMA) and pageable
class BufferJob(Job):
    bb = 65536
    N = 5 * MiB + 12345
    pinned = False
    uses_ctl = True

    def __init__(self, vm, orc, base):
        self.name = "j08_pinned" if self.pinned else "j08_pageable"
        super().__init__(vm, orc, base)
        data = orc.splitmix_bytes(0x801 + self.pinned, self.N)
        self.nb = -(-self.N // self.bb)
        self.offs = np.arange(self.nb, dtype=np.uint64) * self.bb
        self.lens = np.array([_blen(self.N, self.bb, b) for b in range(self.nb)], np.uint32)
        self.prior = orc.hash_blocks(data, self.offs, self.lens)
        self.chosen = [0, 1, 33, self.nb - 1]
        self.new = data.copy()
        for b in self.chosen:
            self.new[b * self.bb] ^= 0xFF
        self.want = orc.hash_blocks(self.new, self.offs, self.lens)

    def stage(self, run):
        s = super().stage(run)
        if self.pinned:
            s["bufs"] = (self.vm.PinnedBuffer(self.N), self.vm.PinnedBuffer(self.N))
            s["src"], s["dst"] = s["bufs"][0].array, s["bufs"][1].array
        else:
            s["src"], s["dst"] = np.empty(self.N, np.uint8), np.empty(self.N, np.uint8)
        s["src"][:] = self.new
        s["dst"][:] = 0xEE
        return s

    def release(self, s):
        for b in s.pop("bufs", ()):
            b.free()
        super().release(s)

    def call(self, s, ctl):
        return self.vm.migrate_buffer(s["src"], s["dst"], self.prior, np.ones(self.nb, np.uint8), block_bytes=self.bb, ctl=ctl)

    def check(self, s, out):
        h, st = out.res
        bad = np.nonzero(h != self.want)[0]
        assert bad.size == 0, bad[:10].tolist()
        dst = s["dst"]
        for b in range(self.nb):
            blk = slice(b * self.bb, b * self.bb + int(self.lens[b]))
            if b in self.chosen:
                assert (dst[blk] == self.new[blk]).all(), b
            else:
                assert (dst[blk] == 0xEE).all(), b           # skipped: left as it was
        assert st["blocks_skipped"] == self.nb - len(self.chosen), st
        assert st["bytes_d2h"] == st["bytes_written"] == int(self.lens[self.chosen].astype(np.uint64).sum()), st


class PinnedBufferJob(BufferJob):
    pinned = True


# 9. an HBM-resident pass: prior, flips and a new length, then one pass
class ResidentJob(Job):
    name = "j09_resident"
    N, BB, SEED = 200, 4 * MiB, 0x909

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        words = self.BB // 8
        blocks = lambda b: orc.splitmix_bytes(self.SEED, self.BB, first_word=b * words)
        self.prior = np.array([orc.xxh64(blocks(b).tobytes()) for b in range(self.N)], np.uint64)
        self.flips = [3, 4, 99, 150, self.N - 1]
        self.valid = np.ones(self.N, np.uint8)
        self.valid[[0, 120]] = 0
        self.short, self.short_len = 77, self.BB - 4097
        self.want = self.prior.copy()
        for b in self.flips:
            x = blocks(b).copy()
            x[:8] ^= 0xFF
            self.want[b] = orc.xxh64(x.tobytes())
        self.want[self.short] = orc.xxh64(blocks(self.short)[:self.short_len].tobytes())
        self.want_surv = sorted(set(self.flips) | {0, 120, self.short})

    def call(self, s, ctl):
        r = self.vm.Resident(self.N, self.BB)
        try:
            r.fill(self.SEED)
            r.set_prior(self.prior, self.valid)
            r.flip(self.flips)
            r.set_len(self.short, self.short_len)
            r.run(1)
            return r.results()
        finally:
            r.close()

    def check(self, s, out):
        h, surv = out.res
        assert surv.tolist() == self.want_surv
        bad = np.nonzero(h != self.want)[0]
        assert bad.size == 0, bad[:10].tolist()


# 11. a plain copy cancelled through its own control once data has been hashed
class CancelJob(Job):
    name, uses_ctl = "j11_cancel", True

    def __init__(self, vm, orc, base):
        super().__init__(vm, orc, base)
        self.src = self.base / "src"
        self.src.mkdir()
        vm.datagen_files(self.src, 0xB11, 4, 64 * MiB)

    def stage(self, run):
        s = super().stage(run)
        (s["dir"] / "dst").mkdir()
        return s

    def call(self, s, ctl):
        stop = threading.Event()

        def canceller():
            while not stop.is_set():
                if ctl.progress()["bytes_hashed"] > 0:
                    ctl.cancel()
                    return
                time.sleep(0.0005)
        t = threading.Thread(target=canceller, daemon=True)
        t.start()
        try:
            return self.vm.migrate_tree(self.src, s["dir"] / "dst", None, s["dir"] / "t.vmig", ctl=ctl)
        finally:
            stop.set()
            t.join()

    def check(self, s, out):
        assert out.err == self.vm.VMIG_ECANCELED, (out.err, out.res)
        assert "cancel" in out.msg and not _foreign(out.msg, self.name), out.msg
        _no_table_left(s["dir"] / "t.vmig")


JOBS = (CopyJob, DiffJob, SnapshotJob, RestoreCorruptJob, ScrubJob, RestorePathsJob, HashBlocksJob, BufferJob,
        PinnedBufferJob, ResidentJob, DiffLanesJob, CancelJob)


def make_jobs(vm, orc, base: Path) -> list:
    return [J(vm, orc, base) for J in JOBS]


def _one(job, s, start=None) -> Outcome:
    vm = job.vm
    ctl = vm.Ctl() if job.uses_ctl else None
    try:
        if start is not None:
            start.wait()
        try:
            res, err, msg = job.call(s, ctl), None, ""
        except vm.VmigError as e:
            res, err, msg = None, e.code, vm.last_error()        # this thread's own text
        return Outcome(res, err, msg, ctl.progress() if ctl else None)
    finally:
        if ctl:
            ctl.close()


def run_alone(jobs) -> list:
    """Each job by itself, one after the other: the counters the mix must reproduce."""
    out = []
    for j in jobs:
        s = j.stage("alone")
        o = _one(j, s)
        check_outcome(j, s, o, None)
        j.release(s)
        out.append(o)
    return out


def run_mix(jobs, run: str, order) -> list:
    """Every job in its own thread, released together by a barrier, started in `order`; returns the outcomes by job."""
    states = [j.stage(run) for j in jobs]
    outs = [None] * len(jobs)
    errors = []
    bar = threading.Barrier(len(jobs))

    def work(i):
        try:
            outs[i] = _one(jobs[i], states[i], bar)
        except BaseException as e:        # noqa: BLE001 -- reported below with the job's name
            errors.append((jobs[i].name, repr(e)))
    th = {i: threading.Thread(target=work, args=(i,), daemon=True) for i in order}
    for i in order:
        th[i].start()
    deadline = time.monotonic() + JOIN_S
    for t in th.values():
        t.join(max(0.0, deadline - time.monotonic()))
    stuck = [jobs[i].name for i, t in th.items() if t.is_alive()]
    assert not stuck, f"calls still waiting after {JOIN_S} s (a pipe was not given back?): {stuck}"
    assert not errors, errors
    return states, outs


def check_outcome(job, s, out, alone):
    """The job's own expectation, the header's progress rule, and the counters of the job run alone."""
    try:
        job.check(s, out)
        st = out.stats()
        if job.progress_is_stats:
            p = out.progress
            assert (p["bytes_total"], p["blocks_total"], p["bytes_written"]) == \
                (st["bytes_total"], st["blocks_total"], st["bytes_written"]), (p, st)
            assert p["bytes_hashed"] + p["bytes_verified"] == st["bytes_h2d"], (p, st)
            assert p["phase_name"] == "DONE" and p["running"] == 0, p
        if alone is not None:
            if st is not None:
                want = alone.stats()
                assert {k: st[k] for k in PINNED} == {k: want[k] for k in PINNED}, (st, want)
            if hasattr(job, "same_as_alone"):
                job.same_as_alone(out, alone)
    except AssertionError as e:
        raise AssertionError(f"{job.name}: {e}") from e


def check_mix(jobs, states, outs, alone):
    for j, s, o, a in zip(jobs, states, outs, alone):
        check_outcome(j, s, o, a)
        j.release(s)


# ------------------------------------------------------------------------------------------ the tests
def test_every_kind_of_call_at_once(vm, orc, shm_tmp):
    """All jobs at once from a barrier (ctypes drops the GIL, so the calls overlap), twice: in job order, then in reverse
    start order so that other pairs overlap.  Each job must match its own oracle and its counters run alone."""
    jobs = make_jobs(vm, orc, shm_tmp)
    alone = run_alone(jobs)
    n = len(jobs)
    for run, order in (("fwd", range(n)), ("rev", range(n - 1, -1, -1))):
        states, outs = run_mix(jobs, run, list(order))
        check_mix(jobs, states, outs, alone)


def _child_one_pipe(a):
    """The engine half of test_one_pipe_serves_every_kind_in_turn: the jobs alone, then at once, all checked here."""
    import __graft_entry__ as g
    from oracle import oracle as orc
    vm = g.load_pkg()
    vm.init(0)
    try:
        jobs = make_jobs(vm, orc, Path(a["base"]))
        alone = run_alone(jobs)
        states, outs = run_mix(jobs, "mix", list(range(len(jobs))))
        check_mix(jobs, states, outs, alone)
        return {"jobs": len(jobs), "launches": {j.name: (o.stats() or {}).get("kernel_launches") for j, o in zip(jobs, outs)}}
    finally:
        vm.shutdown()


def _run_child(fn: str, arg: dict, env: dict, timeout: int = 600) -> dict:
    """test_concurrency.<fn>(arg) in a new Python process with `env` added (the pool settings are read once per process,
    and a new process starts with no lanes in flight).  A child stuck on a leaked pipe is killed at the timeout and fails
    the test."""
    here = Path(__file__).resolve().parent
    code = ("import json, sys; sys.path[:0] = sys.argv[1:3]; import test_concurrency as t; "
            "print(json.dumps(getattr(t, sys.argv[3])(json.loads(sys.argv[4]))))")
    r = subprocess.run([sys.executable, "-c", code, str(here), str(here.parent), fn, json.dumps(arg)],
                       env={**os.environ, **env}, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-6000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("env", [{"VMIG_PIPES_PER_GPU": "1"}, {"VMIG_PIPES_PER_GPU": "1", "VMIG_SLOT_MB": "4", "VMIG_SLOTS": "2"}],
                         ids=["one-pipe", "one-pipe-4MiB-slots"])
def test_one_pipe_serves_every_kind_in_turn(shm_tmp, env):
    """VMIG_PIPES_PER_GPU=1: every call waits for the one pipe (the three-lane call grows the pool to three) and reuses
    slots last used by another kind of call at another block size; with VMIG_SLOT_MB=4 VMIG_SLOTS=2 every 4 MiB block is
    a K1 launch of its own and slots change hands many times."""
    out = _run_child("_child_one_pipe", {"base": str(shm_tmp)}, env)
    assert out["jobs"] == len(JOBS)
    if "VMIG_SLOT_MB" in env:
        assert out["launches"]["j11_cancel"] is None and out["launches"]["j01_copy"] >= 5, out


def _child_pool(a):
    """The engine half of test_pool_is_whole_after_failed_and_cancelled_calls."""
    import __graft_entry__ as g
    from oracle import oracle as orc
    vm = g.load_pkg()
    vm.init(0)
    try:
        idle = [vm.thread_plan(l, 1) for l in (1, 3)]
        jobs = make_jobs(vm, orc, Path(a["base"]))
        states, outs = run_mix(jobs, "mix", list(range(len(jobs))))
        check_mix(jobs, states, outs, [None] * len(jobs))
        after = [vm.thread_plan(l, 1) for l in (1, 3)]
        diff = next(j for j in jobs if type(j) is DiffJob)
        s = diff.stage("after")
        check_outcome(diff, s, _one(diff, s), None)
        diff.release(s)
        return {"idle": idle, "after": after}
    finally:
        vm.shutdown()


def test_pool_is_whole_after_failed_and_cancelled_calls(shm_tmp):
    """In a new process (no lanes in flight), after a mix with a failed and a cancelled call the thread plan is what it was
    before: every pipe checked out was counted back, so later calls are not planned as if others were still running.  A
    fresh diff pass is then right.  VMIG_PLAN_CPUS=64 plans as on a large host, where the plan follows the lanes in flight
    instead of sitting at its floor."""
    out = _run_child("_child_pool", {"base": str(shm_tmp)}, {"VMIG_PLAN_CPUS": "64"})
    assert out["after"] == out["idle"], out


def test_resident_writes_are_ordered_with_the_pass(vm, orc):
    """upload, set_len and set_prior return with their writes done: a pass issued right after, with no other
    synchronisation, hashes the new bytes and lengths against the new prior."""
    n, bb, seed = 64, MiB, 0x5151
    words = bb // 8
    rng = np.random.default_rng(51)
    r = vm.Resident(n, bb)
    try:
        r.fill(seed)
        want = np.array([orc.xxh64(orc.splitmix_bytes(seed, bb, first_word=b * words).tobytes()) for b in range(n)],
                        np.uint64)
        r.set_prior(want, np.ones(n, np.uint8))
        r.run(1)
        h, surv = r.results()
        assert (h == want).all() and surv.size == 0
        for step, b in enumerate((5, 40, 63)):
            data = rng.integers(0, 256, bb - 513 * step, dtype=np.uint8)
            r.upload(b, data)
            r.run(1)
            h, surv = r.results()
            want[b] = orc.xxh64(data.tobytes())
            assert h[b] == want[b] and surv.tolist() == [b], (b, surv)
            assert (r.download(b, data.size) == data).all()
            r.set_prior(want, np.ones(n, np.uint8))
            r.set_len(b, 4096 + step)
            r.run(1)
            h, surv = r.results()
            assert h[b] == orc.xxh64(data[:4096 + step].tobytes()) and surv.tolist() == [b], (b, surv)
            want[b] = h[b]
            valid = np.ones(n, np.uint8)
            valid[[b, (b + 7) % n]] = 0
            r.set_prior(want, valid)
            r.run(1)
            _, surv = r.results()
            assert surv.tolist() == sorted({b, (b + 7) % n}), surv
            r.set_prior(want, np.ones(n, np.uint8))
    finally:
        r.close()
