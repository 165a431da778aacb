"""What one scrub of a snapshot store (vmig_scrub_store) costs next to checking its versions one at a time.

A 10 x 1 GiB layer on tmpfs is snapshotted five times, each version incremental against the one before, with the change
patterns of snapshot_increment.py between them:
  v1 full, v2 unchanged, v3 append (one file grown by 64 MiB), v4 flip30 (30 % of the blocks changed), v5 unchanged
so most of the store is one set of inodes linked by several versions.  Then, alternating, one warm-up and five timed
calls each, in one process on one GPU:
  scrub     one vmig_scrub_store over the five versions
  restores  five checked restores run one after another (vmig_restore_tree, VMIG_F_HASH_ONLY, dst = NULL)
Prints the medians and ranges, bytes_unique and bytes_referenced, and the card's name and power limit.
usage: python profiles/scripts/scrub_store.py [n_files=10] [reps=5]"""
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
    raise SystemExit(f"scrub_store.py: needs ~{3.3 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_scrub_", dir="/dev/shm"))


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
    src = base / "src"
    vm.datagen_files(src, 0x5EED, nf, fb, threads=32)
    pairs = []
    for k, change in enumerate((None, None, append, flip30, None), start=1):
        if change:
            change(src)
        d, t = base / f"v{k}", base / f"v{k}.vmig"
        d.mkdir()
        prev = pairs[-1] if pairs else (None, None)
        s = vm.snapshot_tree(src, d, prev[0], prev[1], t, flags=vm.F_VERIFY)
        print(f"v{k}: written {s['bytes_written'] / 2**20:.0f} MiB, backfilled {s.get('bytes_backfilled', 0) / 2**20:.0f} MiB, "
              f"linked {s.get('files_linked', 0)} files", flush=True)
        pairs.append((d, t))

    def scrub():
        r = vm.scrub_store(pairs, base / "scrub.txt")
        assert r["verdicts"] == [vm.VMIG_OK] * len(pairs), r["verdicts"]
        return r

    def restores():
        h2d = 0
        for d, t in pairs:
            h2d += vm.restore_tree(d, t, None, flags=vm.F_HASH_ONLY)["bytes_h2d"]
        return {"stats": {"bytes_h2d": h2d}}

    calls = {"scrub": scrub, "restores": restores}
    times = {k: [] for k in calls}
    last = {}
    for rep in range(reps + 1):                      # rep 0 warms up both paths
        for name, call in calls.items():
            t0 = time.perf_counter(); r = call(); dt = time.perf_counter() - t0
            print(f"{'warm-up' if rep == 0 else f'rep {rep}':>7} {name:>8}: {dt * 1e3:7.0f} ms  "
                  f"read {r['stats']['bytes_h2d'] / 2**30:6.2f} GiB", flush=True)
            if rep:
                times[name].append(dt)
                last[name] = r
    for name in calls:
        v = times[name]
        print(f"{name}: median {statistics.median(v) * 1e3:.0f} ms ({min(v) * 1e3:.0f}-{max(v) * 1e3:.0f} ms), "
              f"read {last[name]['stats']['bytes_h2d'] / 2**30:.2f} GiB")
    r = last["scrub"]
    print(f"bytes_unique {r['bytes_unique']} ({r['bytes_unique'] / 2**30:.2f} GiB), bytes_referenced {r['bytes_referenced']} "
          f"({r['bytes_referenced'] / 2**30:.2f} GiB), ratio {r['bytes_referenced'] / r['bytes_unique']:.2f}; "
          f"time ratio restores/scrub {statistics.median(times['restores']) / statistics.median(times['scrub']):.2f}")
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
