"""What a compare of a layer with its version snapshot (vmig_compare_snapshot) costs, with and without the layer's own
trusted table, next to the do-it-yourself way: hash the whole layer, then diff the two tables in Python.

The layer on tmpfs is 10 x 1 GiB files plus a config-2B-shaped tree (tools/vmig_datagen layer: log-uniform sizes,
depth-4 tree, symlinks, empty files, a hard-link pair).  It is snapshotted, hashed once (its trusted table), and then one
byte of one 1 GiB file is changed.  Then, alternating, one warm-up and five timed calls each, in one process on one GPU:
  compare        vmig_compare_snapshot without a layer table: every layer file the snapshot has is read
  compare+table  vmig_compare_snapshot with the layer's table: only files whose identity moved are read
  hash+diff      hash_tree of the layer (VMIG_F_HASH_ONLY), then a Python diff of its table with the snapshot's
Prints the medians and ranges, bytes_read and ns_walk, and the card's name and power limit.
usage: python profiles/scripts/compare_snapshot.py [n_files=10] [reps=5] [tree_gib=2] [tree_files=8192]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
import __graft_entry__ as g
from oracle import read_table

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
tree_gib = int(sys.argv[3]) if len(sys.argv) > 3 else 2
tree_files = int(sys.argv[4]) if len(sys.argv) > 4 else 8192
fb = 1 << 30
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
need = 2.2 * (nf + tree_gib) * fb
if st.f_bavail * st.f_frsize < need:
    raise SystemExit(f"compare_snapshot.py: needs ~{need / fb:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_compare_", dir="/dev/shm"))
datagen = ROOT / "tools" / "vmig_datagen"


def table_diff(a, b) -> int:
    """Paths whose (size, block hashes) differ between two block tables, or that only one of them has."""
    ta, tb = read_table(a), read_table(b)
    bb = ta["block_bytes"]

    def per_path(t):
        return {rel: (size, t["hashes"][first:first + -(-size // bb)]) for rel, size, first in t["entries"]}
    pa, pb = per_path(ta), per_path(tb)
    n = 0
    for rel in set(pa) | set(pb):
        x, y = pa.get(rel), pb.get(rel)
        n += x is None or y is None or x[0] != y[0] or not np.array_equal(x[1], y[1])
    return n


try:
    vm.init(1)
    layer, snap = base / "layer", base / "snap"
    layer.mkdir()
    vm.datagen_files(layer / "big", 0x5EED, nf, fb, threads=32)
    if not datagen.exists():
        subprocess.run(["make", "-C", str(ROOT / "tools"), "-s"], check=True)
    subprocess.run([str(datagen), "layer", str(layer / "tree"), "7", str(tree_gib * fb), str(tree_files), "32"], check=True,
                   capture_output=True)
    snap.mkdir()
    vm.snapshot_tree(layer, snap, None, None, base / "snap.vmig")
    vm.hash_tree(layer, base / "layer.vmig")          # the layer's trusted table
    with open(layer / "big" / "f00003.bin", "r+b") as f:
        f.seek(123456789)
        b = f.read(1)
        f.seek(123456789)
        f.write(bytes([b[0] ^ 0xFF]))

    def compare():
        return vm.compare_snapshot(layer, snap, base / "snap.vmig", base / "cmp.txt")

    def compare_table():
        return vm.compare_snapshot(layer, snap, base / "snap.vmig", base / "cmp_t.txt", base / "layer.vmig")

    def hash_diff():
        s = vm.hash_tree(layer, base / "diy.vmig")
        n = table_diff(base / "diy.vmig", base / "snap.vmig")
        return {"stats": s, "bytes_read": s["bytes_h2d"], "paths_changed": n}

    calls = {"compare": compare, "compare+table": compare_table, "hash+diff": hash_diff}
    times = {k: [] for k in calls}
    last = {}
    for rep in range(reps + 1):                      # rep 0 warms up every path
        for name, call in calls.items():
            t0 = time.perf_counter(); r = call(); dt = time.perf_counter() - t0
            print(f"{'warm-up' if rep == 0 else f'rep {rep}':>7} {name:>13}: {dt * 1e3:7.0f} ms  read {r['bytes_read'] / 2**30:6.2f} GiB  "
                  f"walk {r['stats']['ns_walk'] / 1e6:6.1f} ms  paths changed {r['paths_changed']}", flush=True)
            if rep:
                times[name].append(dt)
                last[name] = r
    assert (base / "cmp.txt").read_bytes() == (base / "cmp_t.txt").read_bytes()
    for name in calls:
        v, r = times[name], last[name]
        print(f"{name}: median {statistics.median(v) * 1e3:.0f} ms ({min(v) * 1e3:.0f}-{max(v) * 1e3:.0f} ms), "
              f"bytes_read {r['bytes_read']} ({r['bytes_read'] / 2**30:.2f} GiB), ns_walk {r['stats']['ns_walk'] / 1e6:.1f} ms")
    r = last["compare+table"]
    print(f"compare+table: files_read {r['files_read']}, files_trusted {r['files_trusted']}, findings "
          f"{len((base / 'cmp_t.txt').read_bytes().splitlines())}")
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
