"""The version-sequence model (tests/_layer_model.py) and the reference behaviour it holds the engine to, without a GPU:
the generator is deterministic and covers what it promises, apply + freeze keep a version exactly, expected_written
agrees with a byte comparison, and GNU tar's answer to every kind change at one path is pinned."""
import json
import os
import stat
from pathlib import Path

import pytest

import _layer_model as L
from conftest import make_rich_tree

BB = 65536


def test_script_is_deterministic_and_covers_every_operation_and_kind_pair():
    for seed in range(12):
        s = L.script(seed, 8, BB)
        assert s == L.script(seed, 8, BB) and json.loads(json.dumps(s)) == s, seed
        assert s != L.script(seed + 1, 8, BB)
        assert all(6 <= len(v) <= 12 for v in s), (seed, [len(v) for v in s])
        have = {(o["op"], o.get("var", "")) for v in s for o in v}
        assert [c for c in L.OP_CYCLE if c not in have] == [], seed
        # each pair at its own path, between two consecutive versions: both ends are observed
        first = {}
        for v in s:
            seen = set()
            for o in v:
                if o["op"] == "set_kind":
                    assert o["path"] not in seen, (seed, o)          # one change per path per version
                    seen.add(o["path"])
                    first.setdefault((o["was"], o["kind"]), o["path"])
        assert sorted(first) == sorted(L.KIND_PAIRS_OK), seed
        assert not any(p in L.TAR_REFUSES for p in first), seed
    assert len(L.KIND_PAIRS_OK) == 44 and len(L.TAR_REFUSES) == 5


def _versions(orc, tmp: Path, seed: int, n: int):
    src = tmp / "src"
    L.build_layer(src, orc, BB, make_rich_tree)
    frozen = [tmp / "v0"]
    L.freeze(src, frozen[0])
    ops = L.script(seed, n, BB)
    for k in range(n):
        L.apply(src, ops[k])
        frozen.append(tmp / f"v{k + 1}")
        L.freeze(src, frozen[-1])
        assert orc.compare_trees(src, frozen[-1], mtime_ns=True) == [], (seed, k, json.dumps(ops[k]))
    return src, frozen, ops


def test_apply_and_freeze_round_trip_and_every_kind_pair_happens(orc, shm_tmp):
    src, frozen, ops = _versions(orc, shm_tmp, 3, 8)
    kind_of = lambda root, rel: L.kind_at(os.path.join(root, rel))
    for k, v in enumerate(ops):
        for o in v:
            if o["op"] == "set_kind":
                assert kind_of(frozen[k], o["path"]) == o["was"], (k, o)
                assert kind_of(frozen[k + 1], o["path"]) == o["kind"], (k, o)
    # a frozen version does not move when the layer goes on changing
    assert orc.compare_trees(frozen[0], frozen[1]) != []
    names = {n for _, _, fs in os.walk(os.fsencode(src)) for n in fs}
    assert any(len(n) == 255 for n in names) and any(b"\n" in n for n in names) and any(b"\xff" in n for n in names)


def test_expected_written_agrees_with_a_byte_comparison(orc, shm_tmp):
    _src, frozen, ops = _versions(orc, shm_tmp, 1, 4)
    some_patch = False
    for k in range(1, len(frozen)):
        prev, now = frozen[k - 1], frozen[k]
        mp, mn = L.tree_in_itself(orc, prev), L.tree_in_itself(orc, now)
        second = L.secondaries(mn)
        trusted = L.single_files(mp)
        got = L.expected_written(orc.block_table_of_tree(prev, BB), orc.block_table_of_tree(now, BB), second, trusted, BB)
        n = nbytes = 0
        for rel, r in mn.items():
            rb = os.fsencode(rel)
            if not stat.S_ISREG(r["type"]) or rb in second:
                continue
            new = Path(now, rel).read_bytes()
            old = Path(prev, rel).read_bytes() if rb in trusted else None
            for off in range(0, len(new), BB):
                if old is None or new[off:off + BB] != old[off:off + BB]:      # a shorter or missing slice differs too
                    n += 1
                    nbytes += len(new[off:off + BB])
                else:
                    some_patch = True
        assert got == (n, nbytes), (k, got, (n, nbytes), json.dumps(ops[k - 1]))
    assert some_patch


# ------------------------------------------------------------------------------------------------ what tar does
# The old kind (rows) sits in the destination, the new kind (columns) in the source; the reference's literal pipe runs
# over it.  R: tar replaces the old entry and exits 0.  F: tar fails with exit status 2 and the old entry stays.
#                     file  empty  emptydir  dir  symlink  fifo  hardlink
TAR_MATRIX = {
    "file":     "      R     R       R       R      R       R      R".split(),
    "empty":    "      R     R       R       R      R       R      R".split(),
    "emptydir": "      R     R       R       R      R       R      R".split(),
    "dir":      "      F     F       R       R      F       F      F".split(),
    "symlink":  "      R     R       R       R      R       R      R".split(),
    "fifo":     "      R     R       R       R      R       R      R".split(),
    "hardlink": "      R     R       R       R      R       R      R".split(),
}


def test_the_model_excludes_exactly_what_tar_refuses():
    refused = {(a, b) for a, row in TAR_MATRIX.items() for b, x in zip(L.KINDS, row) if x == "F"}
    assert refused == L.TAR_REFUSES and list(TAR_MATRIX) == list(L.KINDS)


@pytest.mark.parametrize("old", L.KINDS)
def test_tar_outcome_of_every_kind_change_is_pinned(orc, shm_tmp, old):
    for j, new in enumerate(L.KINDS):
        for variant in range(3 if "symlink" in (old, new) else 1):
            src, dst = shm_tmp / f"src_{new}{variant}", shm_tmp / f"dst_{new}{variant}"
            L.kind_tree(dst, old, 30 + variant)
            L.kind_tree(src, new, 61 + variant)
            before = L.kind_at(dst / L.KIND_PATH)
            r = orc.ref_copy(src, dst, check=False)
            if TAR_MATRIX[old][j] == "R":
                assert r.returncode == 0, (old, new, variant, r.stderr)
                # everything the source has is in the destination as the source has it; what else was there stays
                ms, md = orc.tree_manifest(src), orc.tree_manifest(dst)
                assert [k for k in ms if ms[k] != md.get(k)] == [], (old, new, variant)
            else:
                assert r.returncode == 2 and f"{L.KIND_PATH}: Cannot" in r.stderr, (old, new, variant, r.returncode, r.stderr)
                assert L.kind_at(dst / L.KIND_PATH) == before == "dir", (old, new, variant)
