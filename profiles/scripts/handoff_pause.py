"""How long the tenant stays paused in a hand-off: HandoffCopy (the paused pass re-reads the whole layer through
vmig_migrate_tree and re-reads the whole destination to verify it) next to HandoffCopyFromLayer (the paused pass reads
only what the tenant touched since the live pass, through vmig_migrate_layer, and re-reads only what it wrote).

On tmpfs: a layer of 10 x 1 GiB (vmig_datagen) + 10 000 x 4 KiB files.  While pass 1 runs, 0.2 s after it starts, the
tenant rewrites 3 files (1 MiB in place in one 1 GiB file, two 4 KiB files in full) and creates 5 new 4 KiB files.
Alternating, each method hands the same layer over to an empty destination.  Timed with a host clock (every engine call
returns synchronised): pass 1 (start to pause), and the paused pass (pause to return).  Also printed: pass 2's
ns_walk / ns_plan / ns_data / ns_meta / ns_table, bytes_h2d and bytes_read, and the card's name and power limit.
usage: python profiles/scripts/handoff_pause.py [reps=5] [n_big=10] [n_small=10000]"""
import importlib, json, os, shutil, subprocess, sys, tempfile, threading, time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as g

vm = g.load_pkg()
ho = importlib.import_module(vm.__name__ + ".handoff")
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
n_big = int(sys.argv[2]) if len(sys.argv) > 2 else 10
n_small = int(sys.argv[3]) if len(sys.argv) > 3 else 10000
fb, sb = 1 << 30, 4096
card = lambda: subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 2.3 * n_big * fb:
    raise SystemExit(f"handoff_pause.py: needs ~{2.3 * n_big:.0f} GiB free in /dev/shm")
tmp = Path(tempfile.mkdtemp(prefix="vmig_handoff_pause_", dir="/dev/shm"))
try:
    vm.init(1)
    old, new = tmp / "old", tmp / "new"
    old.mkdir()
    vm.datagen_files(old, 7, n_big, fb)
    (old / "small").mkdir()
    rng = np.random.default_rng(5)
    for i in range(n_small):
        (old / "small" / f"s{i:05d}").write_bytes(rng.integers(0, 256, sb, dtype=np.uint8).tobytes())
    big = sorted(p for p in old.iterdir() if p.is_file())
    vm.set_resolver(container_upperdir=lambda n: str({"rs-1": old, "rs-2": new}[n]))
    ho.set_merges_root(tmp)
    methods = {"HandoffCopy": ho.HandoffCopy, "HandoffCopyFromLayer": ho.HandoffCopyFromLayer}
    print(json.dumps({"card": card(), "big_files": n_big, "big_bytes": fb, "small_files": n_small, "small_bytes": sb,
                      "block_bytes": vm.BLOCK_BYTES}), flush=True)
    k = 0
    for rep in range(reps):
        for name, fn in methods.items():
            if new.exists():
                shutil.rmtree(new)
            new.mkdir()
            for p in (tmp / "merges").rglob("blocks.vmig*"):
                p.unlink()
            k += 1

            def tenant(k=k):
                time.sleep(0.2)
                r = np.random.default_rng(100 + k)
                with open(big[k % len(big)], "r+b") as f:
                    f.seek(int(r.integers(0, fb - (1 << 20))))
                    f.write(r.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes())
                for i in (k % n_small, (k * 7 + 1) % n_small):
                    (old / "small" / f"s{i:05d}").write_bytes(r.integers(0, 256, sb, dtype=np.uint8).tobytes())
                for i in range(5):
                    (old / "small" / f"new{k:03d}_{i}").write_bytes(r.integers(0, 256, sb, dtype=np.uint8).tobytes())
            th = threading.Thread(target=tenant)
            t = {}

            def pause(n):
                th.join()                                   # the tenant's writes are done before it is paused
                t["pause"] = time.perf_counter()
            t["start"] = time.perf_counter()
            th.start()
            out = fn("rs-1", "rs-2", pause, lambda n: None)
            t["end"] = time.perf_counter()
            p2 = out["pass2"]
            print(json.dumps({"rep": rep, "method": name, "pass1_seconds": round(t["pause"] - t["start"], 4),
                              "paused_seconds": round(t["end"] - t["pause"], 4), "pass1_error": out["pass1_error"],
                              **{f"pass2_{n[3:]}_seconds": round(p2[n] / 1e9, 4) for n in ("ns_walk", "ns_plan", "ns_data", "ns_meta", "ns_table")},
                              "pass2_bytes_h2d": p2["bytes_h2d"], "pass2_bytes_written": p2["bytes_written"],
                              "pass2_bytes_read": p2.get("bytes_read"), "pass2_files_read": p2.get("files_read"),
                              "pass2_bytes_verified": p2.get("bytes_verified")}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)
finally:
    vm.set_resolver(None, None)
    ho.set_merges_root(None)
    shutil.rmtree(tmp, ignore_errors=True)
