"""What retiring old versions of a snapshot store costs, and what it saves the next incremental snapshot, next to rm -rf.

A 10 x 1 GiB layer on tmpfs is snapshotted eight times (vmig_snapshot_tree, each version incremental against the one
before); versions 2..8 each change one 4 MiB block of one file (file k-2 for version k), so files 7..9 are one inode
linked by all eight versions and file i is shared from version i+2 on.  Then, alternating, one warm-up and `reps` timed
rounds, each on a freshly built store (the store is consumed):
  retire   vmig_retire_versions of v1..v4 keeping v5..v8 (timed), then the next snapshot against v8 (timed)
  rm -rf   shutil.rmtree of v1..v4 and their tables, then the next snapshot against v8 (timed)
For the next snapshot it reports time, bytes_written (ring writes), files_linked and files_base_untrusted.  Then a
keep-last-2 sequence over eight snapshots, once retiring with vmig_retire_versions and once with rm -rf after every
snapshot, reports the total bytes written (ring writes plus base backfill).  Prints the card's name and power limit.
Removing one hard link moves the inode's ctime on Linux tmpfs, ext4 and xfs, and that is what makes rm -rf cost the next
snapshot its base.  Where /dev/shm's unlink does not (some sandboxed filesystems), the script says so and, before each
removal, moves the ctime of the removed versions' files by hand (utime to their own times) as such an unlink would.
usage: python profiles/scripts/retire_store.py [n_files=10] [reps=3]"""
import os, shutil, statistics, subprocess, sys, tempfile, time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import __graft_entry__ as g

vm = g.load_pkg()
nf = int(sys.argv[1]) if len(sys.argv) > 1 else 10
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
fb, BB, NV = 1 << 30, 4 << 20, 8
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip() or "unknown card"
st = os.statvfs("/dev/shm")
if st.f_bavail * st.f_frsize < 4.0 * nf * fb:
    raise SystemExit(f"retire_store.py: needs ~{4.0 * nf:.0f} GiB free in /dev/shm")
base = Path(tempfile.mkdtemp(prefix="vmig_retire_", dir="/dev/shm"))
src = base / "src"


def flip(k: int):
    """Version k's change: one byte of block k of file (k - 2) % nf; applying it twice undoes it."""
    with open(src / f"f{(k - 2) % nf:05d}.bin", "r+b") as f:
        f.seek(k * BB)
        b = f.read(1)
        f.seek(k * BB)
        f.write(bytes([b[0] ^ 0xFF]))


def build(root: Path, keep_last=None, retire=True):
    """The eight versions under root; with keep_last, the older ones are retired (or rm -rf'ed) after each snapshot.
    Leaves src as it found it.  Returns the version pairs still there and the per-snapshot stats."""
    root.mkdir()
    pairs, stats = [], []
    for k in range(1, NV + 1):
        if k > 1:
            flip(k)
        d, t = root / f"v{k}", root / f"v{k}.vmig"
        d.mkdir()
        prev = pairs[-1] if pairs else (None, None)
        stats.append(vm.snapshot_tree(src, d, prev[0], prev[1], t))
        pairs.append((d, t))
        if keep_last and len(pairs) > keep_last:
            old, pairs = pairs[:-keep_last], pairs[-keep_last:]
            as_unlink_would(old)
            if retire:
                vm.retire_versions(old, pairs)
            else:
                for od, ot in old:
                    shutil.rmtree(od)
                    ot.unlink()
    return pairs, stats


def unlink_moves_ctime() -> bool:
    a, b = base / "probe_a", base / "probe_b"
    a.write_bytes(b"x")
    os.link(a, b)
    before = os.stat(a).st_ctime_ns
    time.sleep(0.01)
    b.unlink()
    moved = os.stat(a).st_ctime_ns != before
    a.unlink()
    return moved


def as_unlink_would(old):
    if MOVES:
        return
    for d, _ in old:
        for dp, _dns, fns in os.walk(d):
            for n in fns:
                st = os.lstat(os.path.join(dp, n))
                os.utime(os.path.join(dp, n), ns=(st.st_atime_ns, st.st_mtime_ns))


def unflip():
    for k in range(NV, 1, -1):
        flip(k)


def next_snapshot(root: Path, pairs):
    d = root / "next"
    d.mkdir()
    t0 = time.perf_counter()
    s = vm.snapshot_tree(src, d, pairs[-1][0], pairs[-1][1], root / "next.vmig")
    return time.perf_counter() - t0, s


MOVES = unlink_moves_ctime()
print(f"unlinking one hard link moves the inode's ctime on /dev/shm: {MOVES}"
      + ("" if MOVES else " (the removed versions' files get their ctime moved by hand before each removal)"), flush=True)
try:
    vm.init(1)
    vm.datagen_files(src, 0x5EED, nf, fb, threads=32)
    res = {"retire": [], "rm -rf": []}
    retire_t, retire_last = [], None
    for rep in range(reps + 1):                      # rep 0 warms up both paths
        for arm in ("retire", "rm -rf"):
            root = base / "store"
            pairs, _ = build(root)
            as_unlink_would(pairs[:4])
            if arm == "retire":
                t0 = time.perf_counter()
                r = vm.retire_versions(pairs[:4], pairs[4:])
                dt_r = time.perf_counter() - t0
            else:
                for d, t in pairs[:4]:
                    shutil.rmtree(d)
                    t.unlink()
            dt, s = next_snapshot(root, pairs[4:])
            tag = "warm-up" if rep == 0 else f"rep {rep}"
            extra = f"  (retire {dt_r * 1e3:.0f} ms, re-hashed {r['bytes_rehashed'] / 2**30:.2f} GiB)" if arm == "retire" else ""
            print(f"{tag:>7} {arm:>7}: next snapshot {dt * 1e3:7.0f} ms, written {s['bytes_written'] / 2**30:6.2f} GiB, "
                  f"linked {s['files_linked']}, base untrusted {s['files_base_untrusted']}{extra}", flush=True)
            if rep:
                res[arm].append((dt, s))
                if arm == "retire":
                    retire_t.append(dt_r)
                    retire_last = r
            shutil.rmtree(root)
            unflip()
    for arm, v in res.items():
        ts = [x for x, _ in v]
        s = v[-1][1]
        print(f"next snapshot after {arm}: median {statistics.median(ts) * 1e3:.0f} ms ({min(ts) * 1e3:.0f}-{max(ts) * 1e3:.0f} ms), "
              f"bytes_written {s['bytes_written']} ({s['bytes_written'] / 2**30:.2f} GiB), files_linked {s['files_linked']}, "
              f"files_base_untrusted {s['files_base_untrusted']}")
    r = retire_last
    print(f"retire of 4 of {NV} versions: median {statistics.median(retire_t) * 1e3:.0f} ms ({min(retire_t) * 1e3:.0f}-"
          f"{max(retire_t) * 1e3:.0f} ms); removed {r['entries_removed']} entries, freed {r['bytes_freed'] / 2**30:.2f} GiB; "
          f"{r['records_stale']} records stale, {r['records_restamped']} re-stamped, re-hashed {r['bytes_rehashed'] / 2**30:.2f} GiB, "
          f"{r['tables_rewritten']} tables rewritten")

    for retire in (True, False):
        root = base / "keep2"
        _, stats = build(root, keep_last=2, retire=retire)
        w = sum(s["bytes_written"] for s in stats)
        bf = sum(s["bytes_backfilled"] for s in stats)
        print(f"keep-last-2 over {NV} snapshots with {'retire' if retire else 'rm -rf'}: bytes_written {w} ({w / 2**30:.2f} GiB), "
              f"backfilled {bf / 2**30:.2f} GiB, written + backfilled {(w + bf) / 2**30:.2f} GiB", flush=True)
        shutil.rmtree(root)
        unflip()
    print(f"card: {card}")
finally:
    shutil.rmtree(base, ignore_errors=True)
