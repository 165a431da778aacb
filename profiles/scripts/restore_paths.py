"""What a partial restore (vmig_restore_paths) costs next to a whole checked restore of the same snapshot.

The snapshot, on tmpfs, holds files/ (10 x 1 GiB) and layer/ (a config-2B-shaped layer: tools/vmig_datagen layer, 10 GiB
in 40 960 files, log-uniform 1 KiB-64 MiB, depth-4 tree), with its block table.  Then,
alternating, one warm-up and five timed calls each, in one process on one GPU, each into an emptied destination:
  one_file  vmig_restore_paths of files/f00003.bin (1 GiB)
  one_dir   vmig_restore_paths of layer/a3 (about 1.25 GiB of small files, 5 120 of them)
  whole     vmig_restore_tree of the whole snapshot (20 GiB)
Prints the medians and ranges of the call time, bytes_h2d and ns_walk, and the card's name and power limit.  The claim
under test: the cost of a partial restore follows the selection, not the snapshot.
usage: python profiles/scripts/restore_paths.py [reps=5]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import __graft_entry__ as g

vm = g.load_pkg()
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
GiB = 1 << 30
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 41 * GiB:
    raise SystemExit("restore_paths.py: needs ~41 GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_rpaths_", dir="/dev/shm"))


def empty(d: Path):
    shutil.rmtree(d, ignore_errors=True)
    d.mkdir()


try:
    vm.init(1)
    snap, table, dst = base / "snap", base / "snap.vmig", base / "dst"
    snap.mkdir()
    vm.datagen_files(snap / "files", 0x5EED, 10, GiB, threads=32)
    subprocess.run([str(g.ROOT / "tools" / "vmig_datagen"), "layer", str(snap / "layer"), "2", str(10 * GiB), "40960", "32"],
                   check=True, stdout=subprocess.DEVNULL)
    vm.hash_tree(snap, table)                        # the snapshot's table, hashed on the GPU in place
    n_dir = sum(len(f) for _, _, f in os.walk(snap / "layer" / "a3"))
    print(f"snapshot: {vm.table_info(table)['bytes_total'] / GiB:.2f} GiB, layer/a3: {n_dir} entries", flush=True)

    calls = {
        "one_file": lambda: vm.restore_paths(snap, table, dst, ["files/f00003.bin"]),
        "one_dir": lambda: vm.restore_paths(snap, table, dst, ["layer/a3"]),
        "whole": lambda: vm.restore_tree(snap, table, dst),
    }
    times = {k: [] for k in calls}
    last = {}
    for rep in range(reps + 1):                      # rep 0 warms up every call
        for name, call in calls.items():
            empty(dst)
            t0 = time.perf_counter(); r = call(); dt = time.perf_counter() - t0
            print(f"{'warm-up' if rep == 0 else f'rep {rep}':>7} {name:>8}: {dt * 1e3:8.1f} ms  read {r['bytes_h2d'] / GiB:6.2f} GiB  "
                  f"walk {r['ns_walk'] / 1e6:7.2f} ms", flush=True)
            if rep:
                times[name].append(dt)
                last[name] = r
    for name in calls:
        v, r = times[name], last[name]
        print(f"{name}: median {statistics.median(v) * 1e3:.1f} ms ({min(v) * 1e3:.1f}-{max(v) * 1e3:.1f} ms), "
              f"bytes_total {r['bytes_total']}, bytes_h2d {r['bytes_h2d']} ({r['bytes_h2d'] / GiB:.2f} GiB), "
              f"ns_walk {r['ns_walk'] / 1e6:.2f} ms, files {r['files']}")
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
