"""What an incremental version snapshot costs when the layer's content moved between paths, next to a full one.

A 10 x 1 GiB layer on tmpfs is snapshotted once (v1, verified, the base).  Then, for each of three changes to the
layer, a full verified snapshot and an incremental verified snapshot against v1 are taken into fresh directories,
alternating, one warm-up and five timed calls each, in one process on one GPU:
  renamed        every file moved into a new directory (a checkpoint directory rotated), not a byte changed
  renamed_cp     renamed, plus one file copied to another path with `cp` (a new inode and a new mtime)
  renamed_flip1  renamed (no copy), plus one block changed in every file
For each: wall-time median and range, bytes_written, bytes_d2h, bytes_backfilled, files_linked, and the new space the
snapshot took (tmpfs free blocks before and after the call).  Then the plan-time cost of the base's content index:
ns_plan of a full and of an incremental snapshot of a config-2B-shaped layer (tools/vmig_datagen layer, 40 960 files,
10 GiB) against its own earlier snapshot.  Ends with the card's name and power limit.

The public interface is the one the parent commits have, so the same script measures another build: pass its checkout
as the third argument (it must have been built there).
usage: python profiles/scripts/snapshot_moved.py [n_files=10] [reps=5] [checkout=this one]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
from pathlib import Path

nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
root = Path(sys.argv[3]).resolve() if len(sys.argv) > 3 else Path(__file__).resolve().parents[2]
sys.path.insert(0, str(root))
import __graft_entry__ as g  # noqa: E402

vm = g.load_pkg()
fb, BB = 1 << 30, 4 << 20
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 3.5 * nf * fb:
    raise SystemExit(f"snapshot_moved.py: needs ~{3.5 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_sm_", dir="/dev/shm"))
print(f"build: {root}")


def renamed(src: Path):
    (src / "moved").mkdir()
    for i in range(nf):
        os.rename(src / f"f{i:05d}.bin", src / "moved" / f"f{i:05d}.bin")


def renamed_cp(src: Path):
    subprocess.run(["cp", str(src / "moved" / "f00000.bin"), str(src / "moved" / "copy.bin")], check=True)


def renamed_flip1(src: Path):
    (src / "moved" / "copy.bin").unlink()
    for i in range(nf):
        with open(src / "moved" / f"f{i:05d}.bin", "r+b") as f:
            f.seek(7 * BB)
            w = bytes(x ^ 0xFF for x in f.read(8))
            f.seek(7 * BB)
            f.write(w)


def layer_plan():
    """ns_plan of full and incremental snapshots of a config-2B-shaped layer (the extra lstats and the index)."""
    src, v1 = base / "layer", base / "lv1"
    v1.mkdir()
    subprocess.run([str(root / "tools" / "vmig_datagen"), "layer", str(src), "2", str(10 * fb), "40960", "32"], check=True,
                   capture_output=True)
    vm.snapshot_tree(src, v1, None, None, base / "lv1.vmig", flags=vm.F_VERIFY)
    plans = {"full": [], "incremental": []}
    for rep in range(reps + 1):
        for name, b, t in (("full", None, None), ("incremental", v1, base / "lv1.vmig")):
            dst = base / "ldst"
            shutil.rmtree(dst, ignore_errors=True)
            dst.mkdir()
            s = vm.snapshot_tree(src, dst, b, t, base / "lout.vmig", flags=vm.F_VERIFY)
            if rep:
                plans[name].append(s["ns_plan"] / 1e6)
    for name, v in plans.items():
        print(f"layer 40960 files {name}: ns_plan median {statistics.median(v):.1f} ms ({min(v):.1f}-{max(v):.1f} ms)")


try:
    vm.init(1)
    src, v1 = base / "src", base / "v1"
    v1.mkdir()
    vm.datagen_files(src, 0x5EED, nf, fb, threads=32)
    vm.snapshot_tree(src, v1, None, None, base / "v1.vmig", flags=vm.F_VERIFY)
    calls = {"full": lambda d: vm.snapshot_tree(src, d, None, None, base / "out.vmig", flags=vm.F_VERIFY),
             "incremental": lambda d: vm.snapshot_tree(src, d, v1, base / "v1.vmig", base / "out.vmig", flags=vm.F_VERIFY)}
    for case, change in (("renamed", renamed), ("renamed_cp", renamed_cp), ("renamed_flip1", renamed_flip1)):
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
                if rep:
                    times[name].append(dt)
                    last[name] = (s, grew)
        for name in calls:
            s, grew = last[name]
            v = times[name]
            print(f"{case} {name}: median {statistics.median(v) * 1e3:.0f} ms ({min(v) * 1e3:.0f}-{max(v) * 1e3:.0f} ms), "
                  f"bytes_written {s['bytes_written']}, bytes_d2h {s['bytes_d2h']}, bytes_backfilled {s.get('bytes_backfilled', 0)}, "
                  f"files_linked {s.get('files_linked', 0)}, new space {grew / 2**20:.1f} MiB", flush=True)
    shutil.rmtree(src); shutil.rmtree(v1); shutil.rmtree(base / "dst", ignore_errors=True)
    layer_plan()
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
