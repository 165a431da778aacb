"""Offsets past 4 GiB without a GPU: the metadata pass, the block table and the bindings on a tree that holds one sparse
file of 2^32 + 9 MiB + 777 bytes, and the snapshot backfill copy across 2^32 (tests/backfill_unit.cpp --large).

The plan's block order (tests/plan_unit.cpp), the backfill planning (tests/reuse_unit.cpp) and the scrub reader
(tests/scrub_unit.cpp) have their cases past 2^32 inside those programs, which test_plan_host.py,
test_snapshot_moved_host.py and test_scrub_host.py run.  tests/test_large_offsets.py is the GPU half.

Every expected value is arithmetic on the sizes below or comes from the oracle's table reader."""
import os
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
MiB = 1 << 20
G4 = 1 << 32
BIGF = G4 + 9 * MiB + 777
A_BYTES, Z_BYTES = 3 * 4096 + 5, 70000


def _free_bytes(p) -> int:
    st = os.statvfs(p)
    avail = [st.f_bavail * st.f_frsize]
    for line in Path("/proc/meminfo").read_text().splitlines():
        if line.startswith("MemAvailable:"):
            avail.append(int(line.split()[1]) * 1024)
    return min(avail)


def _sparse_tree(root: Path):
    """a.bin, huge.bin (all hole but its first and last bytes) and z.bin: the walk never reads content."""
    root.mkdir()
    (root / "a.bin").write_bytes(b"a" * A_BYTES)
    with open(root / "huge.bin", "wb") as f:
        f.truncate(BIGF)
        f.write(b"first")
        f.seek(BIGF - 4)
        f.write(b"last")
    (root / "z.bin").write_bytes(b"z" * Z_BYTES)
    assert os.path.getsize(root / "huge.bin") == BIGF


@pytest.mark.parametrize("bb", [4096, 4 * MiB], ids=["4K", "4M"])
def test_manifest_of_a_file_past_4GiB(vm, orc, shm_tmp, bb):
    src, table = shm_tmp / "src", shm_tmp / "m.vmig"
    _sparse_tree(src)
    st = vm.manifest(src, table, block_bytes=bb)
    nb = [-(-n // bb) for n in (A_BYTES, BIGF, Z_BYTES)]
    assert st["bytes_total"] == A_BYTES + BIGF + Z_BYTES and st["bytes_total"] > G4
    assert st["blocks_total"] == sum(nb) and st["files"] == 3
    if bb == 4096:
        assert nb[1] > 1 << 20
    t = orc.read_table(table)
    assert t["block_bytes"] == bb
    assert t["entries"] == [(b"a.bin", A_BYTES, 0), (b"huge.bin", BIGF, nb[0]), (b"z.bin", Z_BYTES, nb[0] + nb[1])]
    assert t["hashes"].size == sum(nb) and not t["hashes"].any()
    info = vm.table_info(table)
    assert info == {"block_bytes": bb, "algo": t["algo"], "n_files": 3, "n_blocks": sum(nb), "bytes_total": st["bytes_total"]}
    assert vm.table_hashes(table).size == sum(nb)


def test_sizes_past_4GiB_cross_the_bindings(vm, shm_tmp):
    src = shm_tmp / "src"
    _sparse_tree(src)
    assert vm.DirSize(src) == A_BYTES + BIGF + Z_BYTES             # the sizes of the entries that are not directories
    assert vm.ToBytes("5GB") == 5 * 1024 ** 3 and vm.ToBytes("4097MB") == 4097 * MiB


def test_backfill_copy_past_4GiB(shm_tmp, tmp_path):
    """copy_range / copy_range_at (csrc/vmig_tree.cpp) between two sparse files: one run longer than 2^32 bytes, then
    separate source and destination offsets above 2^32, through copy_file_range and through pread/pwrite."""
    if _free_bytes(shm_tmp) < 6 << 30:
        pytest.skip("needs ~5 GiB of tmpfs: the copy of a 4 GiB run fills the holes of its output")
    exe = tmp_path / "backfill_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "backfill_unit.cpp"),
                    str(csrc / "vmig_tree.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe), "--large", str(shm_tmp)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "backfill large ok" in r.stdout, r.stdout + r.stderr
    assert os.listdir(shm_tmp) == []
