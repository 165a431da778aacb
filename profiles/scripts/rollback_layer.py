"""What an in-place rollback of a layer to a version snapshot (vmig_rollback_layer) costs next to a pruning restore with
the layer's table as its prior (vmig_restore_tree(..., prior=layer_table, VMIG_F_PRUNE)).

On tmpfs: a 10 x 1 GiB layer made with vmig_datagen, a snapshot of it, and the layer restored from that snapshot with its
own table.  Then 1 % and 10 % of the layer's blocks are changed (one byte each, at offsets scattered over every file) and,
alternating, each method rolls the same layer state back:
  restore           vmig_restore_tree(snap, snap_table, layer, layer_table, layer_table, VMIG_F_PRUNE)
  rollback+table    vmig_rollback_layer(layer, layer_table, snap, snap_table, layer_table)
  rollback          vmig_rollback_layer(layer, NULL, snap, snap_table, layer_table)
The changes are re-applied before each call (outside the timed window); every call returns synchronised.  Prints, per
run, the wall time, bytes_h2d, bytes_written and bytes_fetched, and the card's name and power limit, as JSON lines.
usage: python profiles/scripts/rollback_layer.py [n_files=10] [reps=3]"""
import json, os, shutil, subprocess, sys, tempfile, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
fb, bb = 1 << 30, vm.BLOCK_BYTES
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 2.2 * nf * fb:
    raise SystemExit(f"rollback_layer.py: needs ~{2.2 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_rollback_", dir="/dev/shm"))
try:
    vm.init(1)
    src, snap, layer = base / "src", base / "snap", base / "layer"
    for d in (src, snap, layer):
        d.mkdir()
    vm.datagen_files(src, 7, nf, fb)
    st_, lt = base / "snap.vmig", base / "layer.vmig"
    vm.snapshot_tree(src, snap, None, None, st_)
    shutil.rmtree(src)
    vm.restore_tree(snap, st_, layer, None, lt)
    files = sorted(p for p in layer.iterdir())
    blocks = [(p, b) for p in files for b in range(p.stat().st_size // bb)]

    def mutate(chosen):
        for p, b in chosen:
            st0 = os.stat(p)
            with open(p, "r+b") as f:
                f.seek(b * bb + 4097)
                x = f.read(1)
                f.seek(b * bb + 4097)
                f.write(bytes([x[0] ^ 0x5A]))
            os.utime(p, ns=(st0.st_atime_ns, st0.st_mtime_ns))

    methods = {
        "restore": lambda: vm.restore_tree(snap, st_, layer, lt, lt, flags=vm.F_PRUNE),
        "rollback+table": lambda: vm.rollback_layer(layer, snap, st_, lt, lt),
        "rollback": lambda: vm.rollback_layer(layer, snap, st_, lt, None),
    }
    print(json.dumps({"card": card, "layer_bytes": nf * fb, "block_bytes": bb}), flush=True)
    for frac in (0.01, 0.10):
        rng = np.random.default_rng(11)
        idx = sorted(rng.choice(len(blocks), size=max(1, int(round(frac * len(blocks)))), replace=False))
        chosen = [blocks[i] for i in idx]
        for rep in range(reps):
            for name, fn in methods.items():
                mutate(chosen)
                t0 = time.perf_counter()
                r = fn()
                dt = time.perf_counter() - t0
                s = r["stats"] if "stats" in r else r
                print(json.dumps({"fraction": frac, "blocks_changed": len(chosen), "rep": rep, "method": name, "seconds": round(dt, 4),
                                  "bytes_h2d": s["bytes_h2d"], "bytes_written": s["bytes_written"],
                                  "bytes_fetched": r.get("bytes_fetched"), "bytes_read": r.get("bytes_read")}), flush=True)
    print(json.dumps({"card_after": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                                   capture_output=True, text=True).stdout.strip()}), flush=True)
finally:
    shutil.rmtree(base, ignore_errors=True)
