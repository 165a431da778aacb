"""Content reuse of vmig_snapshot_tree without a GPU: the planning of what a new file takes from which base file and
offset, and the copy with separate source and destination offsets that carries it out (tests/reuse_unit.cpp)."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_reuse_planning_and_offset_copy_unit(shm_tmp, tmp_path):
    exe = tmp_path / "reuse_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "reuse_unit.cpp"),
                    str(csrc / "vmig_reuse.cpp"), str(csrc / "vmig_tree.cpp"), "-o", str(exe)], check=True)
    disk = tmp_path / "disk"
    disk.mkdir()
    r = subprocess.run([str(exe), str(shm_tmp), str(disk)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "reuse unit ok" in r.stdout, r.stdout + r.stderr
