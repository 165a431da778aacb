"""How fast a cancelled call returns, and what polling its progress costs.

A 10 x 1 GiB tree on tmpfs is copied with VMIG_F_VERIFY into a fresh directory, in one process on one GPU:
  latency   a second thread polls the call's control (vmig_ctl_progress) every 0.5 ms and cancels once bytes_hashed
            crosses 10 %, 50 % or 90 % of bytes_total, or once the phase is VERIFY; the time from vmig_ctl_cancel to
            the call's return, median and range of `reps` calls per point (one warm-up call first)
  polling   the plain copy of config 2A (no prior table, no verify) with and without a thread calling vmig_ctl_progress
            every 1 ms, alternating, `reps` calls each: GiB/s of the call
Ends with the card's name and power limit.
usage: python profiles/scripts/cancel_latency.py [n_files=10] [reps=5]"""
import os, shutil, statistics, subprocess, sys, tempfile, threading, time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import __graft_entry__ as g

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
fb = 1 << 30
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 2.2 * nf * fb:
    raise SystemExit(f"cancel_latency.py: needs ~{2.2 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_cl_", dir="/dev/shm"))


def fresh_dst() -> Path:
    d = base / "dst"
    shutil.rmtree(d, ignore_errors=True)
    d.mkdir()
    return d


def cancelled_call(pred):
    """(seconds from the cancel to the return, phase the call stopped in) of one VERIFY copy cancelled when pred holds."""
    dst = fresh_dst()
    with vm.Ctl() as ctl:
        t_cancel = []

        def poll():
            while not t_cancel:
                p = ctl.progress()
                if p["bytes_total"] and pred(p):
                    t_cancel.append(time.perf_counter())
                    ctl.cancel()
                    return
                if p["phase_name"] == "DONE":
                    return
                time.sleep(0.0005)
        th = threading.Thread(target=poll)
        th.start()
        try:
            vm.migrate_tree(base / "src", dst, None, base / "t.vmig", flags=vm.F_VERIFY, ctl=ctl)
            raise SystemExit("cancel_latency.py: the call finished before its cancel point")
        except vm.VmigError as e:
            t_ret = time.perf_counter()
            th.join()
            if e.code != vm.VMIG_ECANCELED:
                raise
            return t_ret - t_cancel[0], vm.PHASES[ctl.progress()["phase"]]


def copy_2a(poll: bool) -> float:
    dst = fresh_dst()
    stop = threading.Event()
    with vm.Ctl() as ctl:
        def poller():
            while not stop.is_set():
                ctl.progress()
                time.sleep(0.001)
        th = threading.Thread(target=poller)
        if poll:
            th.start()
        t0 = time.perf_counter()
        s = vm.migrate_tree(base / "src", dst, None, None, ctl=ctl)
        dt = time.perf_counter() - t0
        stop.set()
        if poll:
            th.join()
    return s["bytes_total"] / dt / 2**30


try:
    vm.init(1)
    vm.datagen_files(base / "src", 0x5EED, nf, fb, threads=32)
    vm.migrate_tree(base / "src", fresh_dst(), None, None, flags=vm.F_VERIFY)          # warm-up: pipes, page cache
    points = [(f"bytes_hashed >= {f:.0%}", lambda p, f=f: p["bytes_hashed"] >= f * p["bytes_total"]) for f in (0.1, 0.5, 0.9)]
    points.append(("phase VERIFY", lambda p: p["phase_name"] == "VERIFY"))
    for name, pred in points:
        lat, phases = [], set()
        for _ in range(reps):
            dt, ph = cancelled_call(pred)
            lat.append(dt * 1e3)
            phases.add(ph)
        print(f"cancel at {name:>20}: median {statistics.median(lat):6.1f} ms, range {min(lat):6.1f}-{max(lat):6.1f} ms "
              f"({reps} calls, stopped in {'/'.join(sorted(phases))})", flush=True)
    copy_2a(False)
    rates = {False: [], True: []}
    for rep in range(reps):
        for poll in (False, True):
            r = copy_2a(poll)
            rates[poll].append(r)
            print(f"2A rep {rep + 1} {'with' if poll else 'without':>7} 1 ms progress polling: {r:6.2f} GiB/s", flush=True)
    for poll in (False, True):
        v = rates[poll]
        print(f"2A {'with' if poll else 'without':>7} polling: median {statistics.median(v):.2f} GiB/s, range "
              f"{min(v):.2f}-{max(v):.2f} GiB/s")
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
