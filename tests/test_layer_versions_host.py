"""CPU side of tests/test_layer_versions.py: what its chain relies on, checked without a GPU.

- A rollback leaves version k as new inodes with whole-second mtimes.  The chain applies the next version's edits to that
  copy, so the script must give the same version k+1 from it as from the original.
- rollback_read restates vmig_rollback_layer's read cost, with the exception include/vmig.h documents: a file the layer
  table vouches for whose extra hard link the prune removes is read.
- The table-write wait (wait_past_recorded_ctimes, tests/table_unit.cpp): a same-size write right after a call records
  a file always moves the file's ctime, on any kernel."""
import os
import shutil
import stat
import struct
import subprocess
import sys
import time
from pathlib import Path

import pytest

import _layer_model as L
from conftest import make_rich_tree
from test_layer_versions import CASES, N, rollback_read

ROOT = Path(__file__).resolve().parent.parent


# ------------------------------------------------------------------------------------------------ the script on a copy
def _rollback_like_copy(src: Path, dst: Path):
    """What a rollback leaves of version k: the same tree as new inodes, every mtime cut to whole seconds."""
    L.freeze(src, dst)
    for dp, dns, fns in os.walk(dst, topdown=False):
        for n in dns + fns + [""]:
            p = os.path.join(dp, n) if n else dp
            st = os.lstat(p)
            s = st.st_mtime_ns // 10**9 * 10**9
            os.utime(p, ns=(s, s), follow_symlinks=False)


def _without_fresh_mtimes(man: dict, since_s: int) -> dict:
    """The edits stamp 'now' on what they touch, at a different moment in each tree: those mtimes are not compared."""
    return {rel: {k: v for k, v in r.items() if not (k == "mtime" and v >= since_s)} for rel, r in man.items()}


@pytest.mark.parametrize("seed", sorted({c[0] for c in CASES}))
def test_script_on_a_rollback_like_copy_gives_the_same_next_version(orc, shm_tmp, seed):
    bb = 4096
    ops = [[]] + L.script(seed, N, bb)
    orig = shm_tmp / "orig"
    L.build_layer(orig, orc, bb, make_rich_tree)
    for k in range(N):
        L.apply(orig, ops[k])
        copy = shm_tmp / f"copy{k}"
        _rollback_like_copy(orig, copy)
        ino = {os.lstat(os.path.join(dp, n)).st_ino for dp, _d, fns in os.walk(copy) for n in fns}
        assert not ino & {os.lstat(os.path.join(dp, n)).st_ino for dp, _d, fns in os.walk(orig) for n in fns}
        nxt = shm_tmp / f"next{k}"
        L.freeze(orig, nxt)
        since = time.time_ns() // 10**9
        L.apply(nxt, ops[k + 1])
        L.apply(copy, ops[k + 1])
        a, b = L.tree_in_itself(orc, nxt), L.tree_in_itself(orc, copy)
        assert L.diff_manifests(_without_fresh_mtimes(a, since), _without_fresh_mtimes(b, since)) == [], (seed, k + 1)
        assert set(a) == set(b)
        shutil.rmtree(copy)
        shutil.rmtree(nxt)


# ------------------------------------------------------------------------------------------------ the rollback's reads
def _table(path: Path, root: Path, records: dict, bb: int = 4096):
    """A format-02 block table naming `records` (rel -> 'ok' | 'stale' | None): the file's identity as it is now, a
    ctime one second off, or no identity.  Hashes are zero: the read rule looks at identities only."""
    files, nb = [], 0
    for rel in sorted(records, key=os.fsencode):
        st = os.lstat(root / rel)
        ino, ct = {"ok": (st.st_ino, st.st_ctime_ns), "stale": (st.st_ino, st.st_ctime_ns + 10**9), None: (0, 0)}[records[rel]]
        files.append((os.fsencode(rel), st.st_size, nb, ino, ct))
        nb += -(-st.st_size // bb)
    raw = bytearray(b"VMIGBT02" + struct.pack("<IIQQ", bb, 1, len(files), nb))
    for rel, size, first, ino, ct in files:
        raw += struct.pack("<I", len(rel)) + rel + struct.pack("<QQQq", size, first, ino, ct)
    path.write_bytes(bytes(raw) + bytes(8 * nb))


def _trees(root: Path, second_path_in_snap: bool):
    layer, snap = root / "layer", root / "snap"
    for d in (layer / "x", layer / "d", snap):
        d.mkdir(parents=True)
    for rel, n in (("a", 5000), ("b", 7000), ("c", 9000), ("sym", 300), ("e", 11)):
        (layer / rel).write_bytes(L.data(len(rel) + n, n))
    (layer / "zero").write_bytes(b"")
    os.link(layer / "a", layer / "x" / "q")                   # x/ is not in the snapshot: the prune removes this link
    os.link(layer / "b", layer / "sym.l")                     # the snapshot has a symlink here: kept by the prune
    if second_path_in_snap:
        os.link(layer / "a", layer / "a2")                    # a path the snapshot has too: compare reads the inode
    for rel, n in (("a", 5000), ("b", 7000), ("c", 9001), ("zero", 0), ("d", 4)):
        (snap / rel).write_bytes(L.data(n, n))                # snapshot content does not matter to the reads
    (snap / "a2").write_bytes(b"x" * 10)
    os.symlink("b", snap / "sym.l")
    (snap / "sym").write_bytes(b"s")
    return layer, snap


def test_rollback_read_with_the_prune_exception(orc, tmp_path):
    layer, snap = _trees(tmp_path / "one", second_path_in_snap=False)
    lt = tmp_path / "one.vmig"
    _table(lt, layer, {"a": "ok", "b": "ok", "c": "stale", "sym": "ok", "zero": "ok", "x/q": None, "e": "ok"})
    size = lambda rel: os.lstat(layer / rel).st_size
    key = lambda rel: (os.lstat(layer / rel).st_dev, os.lstat(layer / rel).st_ino)
    # a: trusted, but its link x/q goes with the prune; b: trusted, its link sym.l stays; c: stale; sym: trusted; d: a
    # directory where the snapshot has a file (pruned); e: only in the layer; zero: no block
    files, nbytes, extra = rollback_read(orc, layer, snap, lt)
    assert extra == {key("a"): size("a")}
    assert (files, nbytes) == (2, size("a") + size("c"))
    # no table: every file both trees have with a block is read, and nothing is an exception
    files, nbytes, extra = rollback_read(orc, layer, snap, None)
    assert extra == {} and (files, nbytes) == (4, size("a") + size("b") + size("c") + size("sym"))


def test_rollback_read_exception_not_counted_twice(orc, tmp_path):
    layer, snap = _trees(tmp_path / "two", second_path_in_snap=True)
    lt = tmp_path / "two.vmig"
    _table(lt, layer, {"a": "ok", "a2": None, "b": "ok", "c": "ok", "sym": "stale"})
    size = lambda rel: os.lstat(layer / rel).st_size
    files, nbytes, extra = rollback_read(orc, layer, snap, lt)
    # a2 has no identity, so the compare reads the inode of a anyway: the prune costs nothing more
    assert extra == {} and (files, nbytes) == (2, size("a") + size("sym"))


# ------------------------------------------------------------------------------------------------ the GPU module
def test_gpu_module_collects_without_a_gpu():
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "tests/test_layer_versions.py"], cwd=ROOT, capture_output=True, text=True, timeout=300)
    ids = sorted(line.split("::", 1)[1] for line in r.stdout.splitlines() if line.startswith("tests/test_layer_versions.py::"))
    want = sorted([f"test_layer_calls_through_nine_versions[seed{c[0]}]" for c in CASES] + ["test_handoff_mirror_over_one_replicaset"])
    assert r.returncode == 0 and ids == want, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------ the table-write wait
def test_write_after_a_recorded_ctime_moves_it_unit(shm_tmp, tmp_path):
    exe = tmp_path / "table_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "table_unit.cpp"),
                    str(csrc / "vmig_table.cpp"), "-o", str(exe)], check=True)
    for work in (shm_tmp, tmp_path):                        # tmpfs, and the disk filesystem of the test directory
        r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 0 and "table unit ok" in r.stdout, r.stdout + r.stderr
