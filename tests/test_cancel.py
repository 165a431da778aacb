"""Cancellable calls with live progress on the GPU (-m gpu): vmig_ctl_* through the Python Ctl.

Every cancel point is chosen from the progress counters: a second thread polls the control until bytes_hashed crosses a
fraction or the phase reaches a value, then cancels once.  After each cancel the call must have returned VMIG_ECANCELED
promptly and left what any failed call leaves (no table, untouched tables and base, a destination a re-run repairs);
expected trees and tables come from the oracle (the literal tar pipe, the C XXH64)."""
import os
import shutil
import subprocess
import sys
import tempfile
import textwrap
import threading
import time
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
BB = 4 * MiB
ROOT = Path(__file__).resolve().parent.parent
PROMPT_S = 3.0                   # generous bound on cancel -> return


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


def _state(root: Path) -> dict:
    """Every entry under root with its kind, content and mtime: what 'untouched' means (as in test_snapshot.py)."""
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for n in [""] + dirnames + filenames:
            p = os.path.join(dirpath, n) if n else dirpath
            st = os.lstat(p)
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[os.path.relpath(p, root)] = (st.st_mode, st.st_mtime_ns, body)
    return out


class Canceller(threading.Thread):
    """Polls ctl.progress() every 0.5 ms; the first time pred(progress) holds it runs action (default ctl.cancel) once."""

    def __init__(self, ctl, pred, action=None):
        super().__init__(daemon=True)
        self.ctl, self.pred, self.action = ctl, pred, action or ctl.cancel
        self.samples, self.t_cancel, self.done = [], None, threading.Event()

    def run(self):
        while not self.done.is_set():
            p = self.ctl.progress()
            self.samples.append(p)
            if self.t_cancel is None and self.pred(p):
                self.t_cancel = time.perf_counter()
                self.action()
                return
            time.sleep(0.0005)


def _run(call, ctl, pred, action=None):
    """call() with a Canceller on ctl; returns (result or VmigError, seconds from the cancel to the return, canceller)."""
    c = Canceller(ctl, pred, action)
    c.start()
    try:
        res = call()
    except Exception as e:       # noqa: BLE001 -- the VmigError is the result under test
        res = e
    t_ret = time.perf_counter()
    c.done.set()
    c.join()
    return res, (None if c.t_cancel is None else t_ret - c.t_cancel), c


def _cancelled(vm, res, latency):
    assert isinstance(res, vm.VmigError) and res.code == vm.VMIG_ECANCELED, res
    assert latency is not None and latency < PROMPT_S, latency


def at_fraction(f):
    return lambda p: p["bytes_total"] and p["bytes_hashed"] >= f * p["bytes_total"]


def in_phase(name):
    return lambda p: p["phase_name"] == name


def _tree(vm, root: Path, n=4, size=256 * MiB, seed=11):
    root.mkdir(parents=True, exist_ok=True)
    vm.datagen_files(root, seed, n, size)
    (root / "sub").mkdir()
    (root / "sub" / "small.txt").write_bytes(b"small\n" * 1000)
    os.symlink("f00000.bin", root / "lnk")
    return root


def _no_table_left(path: Path):
    assert not path.exists(), path
    assert not [n for n in os.listdir(path.parent) if n.startswith(path.name + ".tmp")]


def _matches_oracle(vm, orc, src, dst, table, tmp):
    ref = tmp / "ref"
    shutil.rmtree(ref, ignore_errors=True)
    ref.mkdir()
    orc.ref_copy(src, ref)
    assert orc.compare_trees(ref, dst) == []
    _, want = orc.block_table_of_tree(src)
    assert (vm.table_hashes(table) == want).all()
    shutil.rmtree(ref)


@pytest.fixture(scope="module")
def baseline(vm):
    """Thread plan, thread count and open descriptors once the pipes of a 3-lane call exist."""
    base = Path(tempfile.mkdtemp(prefix="vmig_cancel_base_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    src, dst = _tree(vm, base / "src", n=3, size=16 * MiB), base / "dst"
    dst.mkdir()
    vm.migrate_tree(src, dst, None, base / "t.vmig", lanes_per_gpu=3)
    shutil.rmtree(base)
    return {"plan": [vm.thread_plan(l, 1) for l in (1, 2, 3)], "threads": _threads(), "fds": _fds()}


def _threads():
    return len(os.listdir("/proc/self/task"))


def _fds():
    return len(os.listdir("/proc/self/fd"))


# ---------------------------------------------------------------------------------------------------- 1 + 13: plain copy
@pytest.mark.parametrize("mode", ["1lane", "3lanes", "direct"])
def test_plain_copy_cancelled_at_a_quarter_then_rerun(vm, orc, shm_tmp, baseline, mode):
    """Python Ctl cancelled from a second thread while migrate_tree runs; the same call again repairs the destination."""
    src, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "dst"
    dst.mkdir()
    kw = {"lanes_per_gpu": 3 if mode == "3lanes" else 1, "flags": vm.F_DIRECT_IO if mode == "direct" else 0}
    out = shm_tmp / "t.vmig"
    with vm.Ctl() as ctl:
        res, lat, c = _run(lambda: vm.migrate_tree(src, dst, None, out, ctl=ctl, **kw), ctl, at_fraction(0.25))
        _cancelled(vm, res, lat)
        assert ctl.progress()["running"] == 0 and "DATA" in str(res)
    _no_table_left(out)
    st = vm.migrate_tree(src, dst, None, out, **kw)
    _matches_oracle(vm, orc, src, dst, out, shm_tmp)
    assert st["blocks_total"] == 4 * 64 + 1


# ---------------------------------------------------------------------------------------------------- 2: diff pass
def test_diff_pass_cancelled_keeps_prior_table_and_rerun_copies_touched_files_in_full(vm, orc, shm_tmp, baseline):
    src, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "dst"
    dst.mkdir()
    t1, t2 = shm_tmp / "t1.vmig", shm_tmp / "t2.vmig"
    vm.migrate_tree(src, dst, None, t1)
    for i in range(4):                          # one changed block in every 4 of each file: the diff pass writes
        with open(src / f"f{i:05d}.bin", "r+b") as f:
            for b in range(0, 64, 4):
                f.seek(b * BB + 100)
                f.write(bytes([i + 1]) * 64)
    prior = t1.read_bytes()
    with vm.Ctl() as ctl:
        res, lat, _ = _run(lambda: vm.migrate_tree(src, dst, t1, t2, ctl=ctl), ctl, at_fraction(0.5))
        _cancelled(vm, res, lat)
        wrote = ctl.progress()["bytes_written"]
    assert t1.read_bytes() == prior
    _no_table_left(t2)
    st = vm.migrate_tree(src, dst, t1, t2)
    _matches_oracle(vm, orc, src, dst, t2, shm_tmp)
    if wrote:                                   # a file patched part way no longer matches its table: copied in full
        assert st["files_untrusted"] >= 1, st
    assert st["blocks_skipped"] > 0


# ---------------------------------------------------------------------------------------------------- 3: verify
def test_cancel_in_verify_phase_writes_no_table(vm, shm_tmp, baseline):
    src, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "dst"
    dst.mkdir()
    out = shm_tmp / "t.vmig"
    with vm.Ctl() as ctl:
        res, lat, c = _run(lambda: vm.migrate_tree(src, dst, None, out, flags=vm.F_VERIFY, ctl=ctl), ctl, in_phase("VERIFY"))
        _cancelled(vm, res, lat)
        assert "VERIFY" in str(res), res
    _no_table_left(out)


# ---------------------------------------------------------------------------------------------------- 4: snapshot backfill
def test_snapshot_cancelled_during_backfill_leaves_the_base_intact(vm, orc, shm_tmp, baseline):
    src, v1, v2, v3 = shm_tmp / "src", shm_tmp / "v1", shm_tmp / "v2", shm_tmp / "v3"
    src.mkdir()
    vm.datagen_files(src, 5, 1, 1024 * MiB)
    for d in (v1, v2, v3):
        d.mkdir()
    t1 = shm_tmp / "v1.vmig"
    vm.snapshot_tree(src, v1, None, None, t1)
    ref1 = shm_tmp / "ref1"
    ref1.mkdir()
    orc.ref_copy(src, ref1)
    with open(src / "f00000.bin", "r+b") as f:     # one changed block: the other 255 are copied from the base file
        f.seek(100 * BB)
        f.write(b"\x5a" * 4096)
    before, table_before = _state(v1), t1.read_bytes()
    # every block hashed but the call still in DATA: the last block's writer is copying the rest from the base
    backfill = lambda p: p["phase_name"] == "DATA" and p["blocks_total"] and p["blocks_hashed"] == p["blocks_total"]  # noqa: E731
    with vm.Ctl() as ctl:
        res, lat, _ = _run(lambda: vm.snapshot_tree(src, v2, v1, t1, shm_tmp / "v2.vmig", flags=vm.F_VERIFY, ctl=ctl), ctl, backfill)
        _cancelled(vm, res, lat)
    _no_table_left(shm_tmp / "v2.vmig")
    assert _state(v1) == before and t1.read_bytes() == table_before
    r = shm_tmp / "r1"
    r.mkdir()
    vm.restore_tree(v1, t1, r, None, None, flags=vm.F_VERIFY)
    assert orc.compare_trees(ref1, r) == []
    st = vm.snapshot_tree(src, v3, v1, t1, shm_tmp / "v3.vmig", flags=vm.F_VERIFY)
    assert st["files_backfilled"] == 1
    _matches_oracle(vm, orc, src, v3, shm_tmp / "v3.vmig", shm_tmp)


# ---------------------------------------------------------------------------------------------------- 5: restore
def test_restore_cancelled_is_ecanceled_not_ecorrupt(vm, shm_tmp, baseline):
    src, snap, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "snap", shm_tmp / "dst"
    snap.mkdir(), dst.mkdir()
    t = shm_tmp / "snap.vmig"
    vm.snapshot_tree(src, snap, None, None, t)
    before, tb = _state(snap), t.read_bytes()
    with vm.Ctl() as ctl:
        res, lat, _ = _run(lambda: vm.restore_tree(snap, t, dst, None, shm_tmp / "out.vmig", ctl=ctl), ctl, at_fraction(0.25))
        _cancelled(vm, res, lat)
    _no_table_left(shm_tmp / "out.vmig")
    assert _state(snap) == before and t.read_bytes() == tb


# ---------------------------------------------------------------------------------------------------- 6: move
@pytest.mark.parametrize("phase", ["DATA", "UNLINK"])
def test_move_is_intact_or_complete(vm, orc, shm_tmp, baseline, phase):
    src, dst, ref = _tree(vm, shm_tmp / "src", n=2), shm_tmp / "dst", shm_tmp / "ref"
    many = src / "many"
    many.mkdir()
    for i in range(3000):                       # enough entries for the unlink phase to be seen
        (many / f"e{i:05d}").write_bytes(b"%d\n" % i)
    dst.mkdir(), ref.mkdir()
    orc.ref_copy(src, ref)
    before = orc.tree_manifest(src)
    with vm.Ctl() as ctl:
        pred = at_fraction(0.25) if phase == "DATA" else in_phase("UNLINK")
        res, lat, c = _run(lambda: vm.migrate_tree(src, dst, None, None, flags=vm.MOVE_DIR_FLAGS, ctl=ctl), ctl, pred)
    if isinstance(res, vm.VmigError):
        assert res.code == vm.VMIG_ECANCELED and lat < PROMPT_S, res
        assert orc.tree_manifest(src) == before
    else:
        assert os.listdir(src) == [] and orc.compare_trees(ref, dst) == []
    if phase == "DATA":
        assert isinstance(res, vm.VmigError), "a cancel at a quarter of the data pass must be honoured"


# ---------------------------------------------------------------------------------------------------- 7: pipe wait
def test_call_waiting_for_a_pipe_is_cancelled(shm_tmp):
    """VMIG_PIPES_PER_GPU=1 is read once per process: a child process.  The second call waits for the only pipe, is
    cancelled while it waits, returns VMIG_ECANCELED while the first still runs, and the first call's copy is right."""
    script = textwrap.dedent(f"""
        import sys, threading, time
        sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
        import __graft_entry__ as g
        from pathlib import Path
        from oracle import oracle as orc
        vm = g.load_pkg(); vm.init(0)
        base = Path({str(shm_tmp)!r})
        src, d1, d2 = base / "src", base / "d1", base / "d2"
        for d in (src, d1, d2): d.mkdir()
        vm.datagen_files(src, 3, 8, 256 << 20)
        first = {{}}
        with vm.Ctl() as c1, vm.Ctl() as c2:
            t = threading.Thread(target=lambda: first.update(st=vm.migrate_tree(src, d1, None, base / "t1.vmig", ctl=c1)))
            t.start()
            while c1.progress()["bytes_hashed"] == 0: time.sleep(0.0005)
            err = {{}}
            def second():
                try: vm.migrate_tree(src, d2, None, None, ctl=c2)
                except vm.VmigError as e: err["code"] = e.code; err["msg"] = str(e)
            t2 = threading.Thread(target=second); t2.start()
            while c2.progress()["phase_name"] != "DATA": time.sleep(0.0005)
            time.sleep(0.01)
            assert c2.progress()["bytes_hashed"] == 0 and c1.progress()["running"] == 1
            t0 = time.perf_counter(); c2.cancel(); t2.join(); lat = time.perf_counter() - t0
            first_running = c1.progress()["running"]
            t.join()
        assert err["code"] == vm.VMIG_ECANCELED and "staging pipe" in err["msg"], err
        ref = base / "ref"; ref.mkdir(); orc.ref_copy(src, ref)
        assert orc.compare_trees(ref, d1) == []
        _, want = orc.block_table_of_tree(src)
        assert (vm.table_hashes(base / "t1.vmig") == want).all()
        print(f"pipe wait ok: cancelled in {{lat * 1e3:.1f}} ms, first call still running: {{first_running}}")
        assert lat < 1.0
    """)
    env = dict(os.environ, VMIG_PIPES_PER_GPU="1")
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "pipe wait ok" in r.stdout, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------- 8: buffer
def test_migrate_buffer_cancelled_leaves_unwritten_regions(vm, baseline):
    n = 1024 * MiB
    src = np.frombuffer(np.random.default_rng(3).bytes(n), dtype=np.uint8)
    dst = np.full(n, 0xEE, dtype=np.uint8)
    with vm.Ctl() as ctl:
        res, lat, _ = _run(lambda: vm.migrate_buffer(src, dst, ctl=ctl), ctl, at_fraction(0.25))
        _cancelled(vm, res, lat)
        written = ctl.progress()["bytes_written"]
    s, d = src.reshape(-1, BB), dst.reshape(-1, BB)
    same = (s == d).all(axis=1)
    untouched = (d == 0xEE).all(axis=1)
    assert (same | untouched).all()                 # every block is either written whole or untouched
    assert int(same.sum()) * BB == written and not same.all()


# ---------------------------------------------------------------------------------------------------- 9: progress
def test_progress_is_monotonic_ordered_and_ends_equal_to_stats(vm, orc, shm_tmp, baseline):
    src, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "dst"
    dst.mkdir()
    out = shm_tmp / "t.vmig"
    with vm.Ctl() as ctl:
        res, _, c = _run(lambda: vm.migrate_tree(src, dst, None, out, flags=vm.F_VERIFY, ctl=ctl), ctl, lambda p: False)
        final = ctl.progress()
    assert isinstance(res, dict), res
    keys = ("bytes_total", "blocks_total", "bytes_hashed", "blocks_hashed", "bytes_written", "bytes_verified")
    for a, b in zip(c.samples, c.samples[1:]):
        assert all(a[k] <= b[k] for k in keys), (a, b)
    order = ["IDLE", "WALK", "PRUNE", "DATA", "META", "VERIFY", "TABLE", "UNLINK", "DONE"]
    seen = [p["phase_name"] for p in c.samples] + [final["phase_name"]]
    idx = [order.index(s) for s in seen]
    assert idx == sorted(idx), seen
    assert "DATA" in seen and final["phase_name"] == "DONE" and final["running"] == 0
    assert final["bytes_total"] == res["bytes_total"] and final["blocks_total"] == res["blocks_total"]
    assert final["bytes_written"] == res["bytes_written"]
    assert final["bytes_hashed"] + final["bytes_verified"] == res["bytes_h2d"]
    assert final["blocks_hashed"] == res["blocks_total"] and final["bytes_verified"] == final["bytes_hashed"]
    _matches_oracle(vm, orc, src, dst, out, shm_tmp)


# ---------------------------------------------------------------------------------------------------- 10: state after
def test_state_after_the_cancels_is_back_to_baseline(vm, orc, shm_tmp, baseline):
    assert [vm.thread_plan(l, 1) for l in (1, 2, 3)] == baseline["plan"]
    assert _threads() == baseline["threads"], (_threads(), baseline["threads"])
    assert _fds() == baseline["fds"], (_fds(), baseline["fds"])
    src, dst = _tree(vm, shm_tmp / "src", n=2, size=64 * MiB), shm_tmp / "dst"
    dst.mkdir()
    vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", lanes_per_gpu=3)
    _matches_oracle(vm, orc, src, dst, shm_tmp / "t.vmig", shm_tmp)


# ---------------------------------------------------------------------------------------------------- 11: shutdown
def test_shutdown_during_a_call_cancels_it_and_waits(vm, orc, shm_tmp):
    src, dst = _tree(vm, shm_tmp / "src"), shm_tmp / "dst"
    dst.mkdir()
    done = {}

    def shut():
        vm.shutdown()
        done["t"] = time.perf_counter()
    with vm.Ctl() as ctl:
        res, lat, c = _run(lambda: vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", ctl=ctl), ctl, at_fraction(0.25),
                           action=lambda: threading.Thread(target=shut).start())
        _cancelled(vm, res, lat)
        while "t" not in done:
            time.sleep(0.001)
    assert done["t"] >= c.t_cancel + lat - 0.01            # shutdown returned only after the call had returned
    _no_table_left(shm_tmp / "t.vmig")
    vm.init(0)
    vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig")
    _matches_oracle(vm, orc, src, dst, shm_tmp / "t.vmig", shm_tmp)


# ---------------------------------------------------------------------------------------------------- 12: hand-off budget
def _handoff(vm):
    import importlib
    return importlib.import_module(vm.__name__ + ".handoff")


def test_handoff_pause_budget(vm, orc, shm_tmp):
    ho = _handoff(vm)
    old, new = shm_tmp / "upper_old", shm_tmp / "upper_new"
    old.mkdir(), new.mkdir()
    vm.datagen_files(old, 9, 4, 256 * MiB)
    calls = []
    vm.set_resolver(container_upperdir=lambda n: str({"rs-1": old, "rs-2": new}[n]))
    ho.set_merges_root(shm_tmp)
    try:
        before = _state(old)
        with pytest.raises(vm.VmigError) as ei:
            ho.HandoffCopy("rs-1", "rs-2", lambda n: calls.append(("pause", n)), lambda n: calls.append(("resume", n)),
                           pauseBudget=0.005)
        assert ei.value.code == vm.VMIG_ECANCELED and getattr(ei.value, "pause_budget_exceeded", False), ei.value
        assert calls == [("pause", "rs-1"), ("resume", "rs-1")]
        assert _state(old) == before
        vdir = shm_tmp / "merges" / "rs" / "rs-2"
        assert not (vdir / "blocks.vmig").exists() and not (vdir / "blocks.vmig.pass1").exists()
        assert not [n for n in os.listdir(vdir) if ".tmp" in n]
        # budget 0: no limit, today's behaviour
        calls.clear()
        out = ho.HandoffCopy("rs-1", "rs-2", lambda n: calls.append(("pause", n)), lambda n: calls.append(("resume", n)),
                             pauseBudget=0)
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
