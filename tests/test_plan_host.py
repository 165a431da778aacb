"""The plan of a tree call without a GPU: block order, in-place and base trust, prior hashes and the cancel check of
csrc/vmig_plan.cpp on real files (tests/plan_unit.cpp)."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_tree_plan_unit(shm_tmp, tmp_path):
    exe = tmp_path / "plan_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "plan_unit.cpp"),
                    str(csrc / "vmig_plan.cpp"), str(csrc / "vmig_tree.cpp"), str(csrc / "vmig_table.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe), str(shm_tmp)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "plan unit ok" in r.stdout, r.stdout + r.stderr
