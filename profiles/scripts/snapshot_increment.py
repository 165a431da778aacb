"""What an incremental version snapshot (vmig_snapshot_tree against the previous snapshot) costs next to a full one.

A 10 x 1 GiB layer on tmpfs is snapshotted once (v1, the base).  Then, for each of three changes to the layer, a full
verified snapshot and an incremental verified snapshot against v1 are taken into fresh directories, alternating, one
warm-up and five timed calls each, in one process on one GPU:
  unchanged  the layer as v1 holds it
  append     one file grown by 64 MiB
  flip30     30 % of the blocks changed (config 4's mutation: the first 8 bytes of each picked block XORed with 0xFF),
             so every file changes and every file is backfilled
For each: wall-time median and spread, bytes_written, bytes_d2h, bytes_backfilled, files_linked, and the new space the
snapshot took (tmpfs free blocks before and after the call).  Ends with the card's name and power limit.
usage: python profiles/scripts/snapshot_increment.py [n_files=10] [reps=5]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import __graft_entry__ as g

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
fb, BB = 1 << 30, 4 << 20
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 3.3 * nf * fb:
    raise SystemExit(f"snapshot_increment.py: needs ~{3.3 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_si_", dir="/dev/shm"))


def flip30(src: Path):
    per_file = fb // BB
    rng = np.random.default_rng(44)
    for b in sorted(rng.choice(nf * per_file, nf * per_file * 3 // 10, replace=False)):
        with open(src / f"f{b // per_file:05d}.bin", "r+b") as f:
            f.seek(int(b % per_file) * BB)
            w = bytes(x ^ 0xFF for x in f.read(8))
            f.seek(int(b % per_file) * BB)
            f.write(w)


def append(src: Path):
    with open(src / "f00003.bin", "ab") as f:
        f.write(np.full(64 << 20, 0xA5, dtype=np.uint8).tobytes())


try:
    vm.init(1)
    src, v1 = base / "src", base / "v1"
    v1.mkdir()
    vm.datagen_files(src, 0x5EED, nf, fb, threads=32)
    vm.snapshot_tree(src, v1, None, None, base / "v1.vmig", flags=vm.F_VERIFY)
    calls = {"full": lambda d: vm.snapshot_tree(src, d, None, None, base / "out.vmig", flags=vm.F_VERIFY),
             "incremental": lambda d: vm.snapshot_tree(src, d, v1, base / "v1.vmig", base / "out.vmig", flags=vm.F_VERIFY)}
    for case, change in (("unchanged", None), ("append", append), ("flip30", flip30)):
        if change:
            change(src)
        times = {k: [] for k in calls}
        last = {}
        for rep in range(reps + 1):                  # rep 0 warms up both paths
            for name, call in calls.items():
                dst = base / "dst"
                shutil.rmtree(dst, ignore_errors=True)
                dst.mkdir()
                f0 = os.statvfs(base).f_bfree
                t0 = time.perf_counter(); s = call(dst); dt = time.perf_counter() - t0
                grew = (f0 - os.statvfs(base).f_bfree) * os.statvfs(base).f_frsize
                print(f"{case:>9} {'warm-up' if rep == 0 else f'rep {rep}':>7} {name:>11}: {dt * 1e3:7.0f} ms  "
                      f"written {s['bytes_written'] / 2**20:8.0f} MiB  d2h {s['bytes_d2h'] / 2**20:8.0f} MiB  "
                      f"backfilled {s.get('bytes_backfilled', 0) / 2**20:8.0f} MiB  linked {s.get('files_linked', 0):2d} files  "
                      f"new space {grew / 2**20:8.1f} MiB", flush=True)
                if rep:
                    times[name].append(dt)
                    last[name] = (s, grew)
        spread = lambda v: (max(v) - min(v)) / statistics.median(v) * 100      # noqa: E731
        for name in calls:
            s, grew = last[name]
            print(f"{case} {name}: median {statistics.median(times[name]) * 1e3:.0f} ms (spread {spread(times[name]):.1f} %, "
                  f"{min(times[name]) * 1e3:.0f}-{max(times[name]) * 1e3:.0f} ms), bytes_written {s['bytes_written']}, "
                  f"bytes_d2h {s['bytes_d2h']}, bytes_backfilled {s.get('bytes_backfilled', 0)}, "
                  f"files_linked {s.get('files_linked', 0)}, new space {grew / 2**20:.1f} MiB")
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
