"""Every option flag and environment variable the engine reads is exercised by tests/test_settings.py or named on its
EXEMPT list with a reason (CPU only: reads sources, runs nothing).

A setting added to include/vmig.h or read with env_long()/getenv() under csrc/ (the probes excepted) fails this test
until test_settings.py turns it -- under its VMIG_* name in a string, or as vm.F_* for a flag -- or says why not."""
import ast
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SETTINGS = Path(__file__).resolve().parent / "test_settings.py"


def engine_names() -> set:
    flags = set(re.findall(r"^#define\s+(VMIG_F_[A-Z0-9_]+)\s", (ROOT / "include" / "vmig.h").read_text(), re.M))
    env = set()
    for p in sorted((ROOT / "gpu-docker-api_b200" / "csrc").rglob("*")):
        if p.suffix in (".cu", ".cpp", ".h", ".cuh") and "probe" not in p.relative_to(ROOT).parts:
            env |= set(re.findall(r"\b(?:env_long|getenv)\(\s*\"(VMIG_[A-Z0-9_]+)\"", p.read_text()))
    return flags | env


def exercised_and_exempt():
    """(names test_settings.py uses outside EXEMPT, EXEMPT's reasons)."""
    tree = ast.parse(SETTINGS.read_text())
    exempt, used = {}, set()
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "EXEMPT" for t in node.targets):
            exempt = ast.literal_eval(node.value)
            continue
        docs = {id(n.value) for n in ast.walk(node) if isinstance(n, ast.Expr) and isinstance(n.value, ast.Constant)}
        for n in ast.walk(node):
            if id(n) in docs:
                continue                    # a docstring names a setting, it does not turn it
            if isinstance(n, ast.Constant) and isinstance(n.value, str):
                used |= set(re.findall(r"\bVMIG_[A-Z0-9_]+", n.value)) | {"VMIG_" + f for f in re.findall(r"\b(F_[A-Z0-9_]+)\b", n.value)}
            elif isinstance(n, ast.Attribute) and n.attr.startswith("F_"):
                used.add("VMIG_" + n.attr)
    return used, exempt


def test_engine_names_are_found():
    names = engine_names()
    assert {"VMIG_F_MTIME_NS", "VMIG_F_NO_METADATA", "VMIG_SLOT_MB", "VMIG_WALK_THREADS", "VMIG_RING_OUT_NODE",
            "VMIG_BIND_WRITERS", "VMIG_LANES_PER_GPU", "VMIG_DIRECT_IO"} <= names, sorted(names)


def test_every_setting_is_exercised_or_exempt():
    used, exempt = exercised_and_exempt()
    missing = sorted(engine_names() - used - set(exempt))
    assert missing == [], f"neither exercised in tests/test_settings.py nor on its EXEMPT list: {missing}"


def test_exemptions_are_few_and_give_a_reason():
    used, exempt = exercised_and_exempt()
    assert len(exempt) <= 12, sorted(exempt)
    assert all(isinstance(r, str) and len(r) >= 20 for r in exempt.values()), exempt
    assert not set(exempt) - engine_names(), sorted(set(exempt) - engine_names())     # no stale exemption
    assert not set(exempt) & used, sorted(set(exempt) & used)                           # exempt means not turned
