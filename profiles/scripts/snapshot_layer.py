"""What a version snapshot taken through the layer's own block table (vmig_snapshot_layer) costs next to one that reads
the whole layer (vmig_snapshot_tree), both against the same base snapshot.

On tmpfs: a 10 x 1 GiB layer made with vmig_datagen, a snapshot of it (the base), and the layer put back from that
snapshot.  Then 1 % (later 10 %) of the layer's blocks are changed (one byte each, at offsets scattered over every file,
mtimes kept), one new 64 MiB file is added, and the layer's table is written by a hash-only migration of the layer (the
table a hand-off leaves: it vouches for every file as it now is).  Alternating, each method snapshots that layer state
into a new directory:
  tree+verify     vmig_snapshot_tree(layer, dst, base, base_table, out, VMIG_F_VERIFY)
  layer+verify    vmig_snapshot_layer(layer, layer_table, dst, base, base_table, out, VMIG_F_VERIFY)
  tree            vmig_snapshot_tree(..., 0)
  layer           vmig_snapshot_layer(..., 0)
After each call the new version is retired with vmig_retire_versions (outside the timed window), which re-stamps the
base records its links left stale, so every call sees the same trusted base.  Every call returns synchronised.  Prints,
per run, the wall time, bytes_h2d, bytes_written and bytes_read, and the card's name and power limit, as JSON lines.
usage: python profiles/scripts/snapshot_layer.py [n_files=10] [reps=2]"""
import json, os, shutil, subprocess, sys, tempfile, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
fb, bb = 1 << 30, vm.BLOCK_BYTES
card = lambda: subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 2.5 * nf * fb:
    raise SystemExit(f"snapshot_layer.py: needs ~{2.5 * nf:.0f} GiB free in /dev/shm")
tmp = Path(tempfile.mkdtemp(prefix="vmig_snaplayer_", dir="/dev/shm"))
try:
    vm.init(1)
    src, base, layer = tmp / "src", tmp / "base", tmp / "layer"
    for d in (src, base, layer):
        d.mkdir()
    vm.datagen_files(src, 7, nf, fb)
    bt, lt = tmp / "base.vmig", tmp / "layer.vmig"
    vm.snapshot_tree(src, base, None, None, bt)
    shutil.rmtree(src)
    vm.restore_tree(base, bt, layer, None, None)
    files = sorted(layer.iterdir())
    blocks = [(p, b) for p in files for b in range(p.stat().st_size // bb)]

    def flip(chosen):
        for p, b in chosen:
            st0 = os.stat(p)
            with open(p, "r+b") as f:
                f.seek(b * bb + 4097)
                x = f.read(1)
                f.seek(b * bb + 4097)
                f.write(bytes([x[0] ^ 0x5A]))
            os.utime(p, ns=(st0.st_atime_ns, st0.st_mtime_ns))

    dst, out = tmp / "dst", tmp / "dst.vmig"
    methods = {
        "tree+verify": lambda: vm.snapshot_tree(layer, dst, base, bt, out, flags=vm.F_VERIFY),
        "layer+verify": lambda: vm.snapshot_layer(layer, dst, base, bt, out, lt, flags=vm.F_VERIFY),
        "tree": lambda: vm.snapshot_tree(layer, dst, base, bt, out),
        "layer": lambda: vm.snapshot_layer(layer, dst, base, bt, out, lt),
    }
    print(json.dumps({"card": card(), "layer_bytes": nf * fb, "block_bytes": bb}), flush=True)
    for frac in (0.01, 0.10):
        rng = np.random.default_rng(11)
        idx = sorted(rng.choice(len(blocks), size=max(1, int(round(frac * len(blocks)))), replace=False))
        chosen = [blocks[i] for i in idx]
        flip(chosen)
        (layer / "new.bin").write_bytes(np.random.default_rng(12).integers(0, 256, 64 << 20, dtype=np.uint8).tobytes())
        vm.hash_tree(layer, lt)
        for rep in range(reps):
            for name, fn in methods.items():
                dst.mkdir()
                t0 = time.perf_counter()
                r = fn()
                dt = time.perf_counter() - t0
                print(json.dumps({"fraction": frac, "blocks_changed": len(chosen), "rep": rep, "method": name, "seconds": round(dt, 4),
                                  "bytes_h2d": r["bytes_h2d"], "bytes_written": r["bytes_written"], "bytes_read": r.get("bytes_read"),
                                  "files_linked": r["files_linked"], "bytes_backfilled": r["bytes_backfilled"]}), flush=True)
                vm.retire_versions([(dst, out)], [(base, bt)])
        flip(chosen)                                   # the same byte flipped back: the layer holds the base's bytes again
        (layer / "new.bin").unlink()
    print(json.dumps({"card_after": card()}), flush=True)
finally:
    shutil.rmtree(tmp, ignore_errors=True)
