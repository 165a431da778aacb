"""What the snapshot check of vmig_restore_tree costs over vmig_migrate_tree: the same 10 x 1 GiB tmpfs snapshot is
copied by migrate_tree and by restore_tree (checked against its block table) into fresh destinations, alternating, in
one process on one GPU.  Prints every call's time, the median of each, and the card's name and power limit.
usage: python profiles/scripts/restore_overhead.py [n_files=10] [reps=5]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
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
if st.f_bavail * st.f_frsize < 2.5 * nf * fb:
    raise SystemExit(f"restore_overhead.py: needs ~{2.5 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_ro_", dir="/dev/shm"))
try:
    vm.init(1)
    vm.datagen_files(base / "snap", 0x5EED, nf, fb, threads=32)
    table = base / "snap.vmig"
    vm.hash_tree(base / "snap", table)
    calls = {"migrate": lambda d: vm.migrate_tree(base / "snap", d, None, base / "out.vmig"),
             "restore": lambda d: vm.restore_tree(base / "snap", table, d, None, base / "out.vmig")}
    times = {k: [] for k in calls}
    for rep in range(reps + 1):                  # rep 0 warms up both paths
        for name, call in calls.items():
            dst = base / "dst"
            shutil.rmtree(dst, ignore_errors=True)
            dst.mkdir()
            t0 = time.perf_counter(); s = call(dst); dt = time.perf_counter() - t0
            assert (vm.table_hashes(base / "out.vmig") == vm.table_hashes(table)).all()
            print(f"{'warm-up' if rep == 0 else f'rep {rep}':>7} {name}: {dt * 1e3:7.0f} ms  "
                  f"{nf * fb / dt / (1 << 30):6.2f} GiB/s  ({s['blocks_total']} blocks, {s['lanes_used']} lanes)", flush=True)
            if rep:
                times[name].append(dt)
    m, r = statistics.median(times["migrate"]), statistics.median(times["restore"])
    spread = lambda v: (max(v) - min(v)) / statistics.median(v) * 100      # noqa: E731
    print(f"median migrate {m * 1e3:.0f} ms (spread {spread(times['migrate']):.1f} %), restore {r * 1e3:.0f} ms "
          f"(spread {spread(times['restore']):.1f} %): restore/migrate = {r / m:.3f}; card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
