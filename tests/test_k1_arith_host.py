"""The CPU model of K1's 32-bit round (tests/_k1_chain.py) and the edge-driven blocks it builds, against the oracle.

The model must equal the oracle, the built blocks must put every edge class of the round in every lane at every
scheduled position, and three variants of the round that each drop one rare carry or cross term must disagree with
the oracle on the built blocks while agreeing with it on the random blocks the GPU suite hashes today: those inputs
cannot tell such a slip from the kernel as written, the built ones can.  tests/test_k1_arith.py hashes the built
blocks on the GPU."""
import numpy as np
import pytest

import _k1_chain as K
from test_gpu import ring_boundary_case

KiB = 1024
# 1 KiB = one chunk; 7 chunks + a 13-byte tail; 8 chunks and a ragged 17-stripe chunk + 31 tail bytes; 2 stripes; 1
LENGTHS = [KiB, 7 * KiB + 13, 8 * KiB + 544 + 31, 64, 32]
SEED = 0xC4A1


@pytest.fixture(scope="module")
def built():
    blocks = K.built_blocks(LENGTHS, SEED)
    buf, offs, lens = K.pack([b for _n, _ph, b, _miss in blocks], SEED)
    return blocks, buf, offs, lens


def test_model_equals_oracle_on_random_blocks(orc):
    rng = np.random.default_rng(0x7A)
    lens = np.array(list(range(0, 97)) + [1023, 1024, 1025, 1056, 6 * KiB + 33, 65536 + 7], np.uint32)
    offs = np.cumsum(np.concatenate([[3], lens[:-1].astype(np.uint64) + rng.integers(1, 9, lens.size - 1)])).astype(np.uint64)
    buf = rng.integers(0, 256, int(offs[-1] + lens[-1]), dtype=np.uint8)
    want = orc.hash_blocks(buf, offs, lens)
    assert (K.model_hashes(buf, offs, lens) == want).all()
    _t_in, _m, _t_out, _first, plain = K.plain_rounds(buf, offs, lens)
    assert (plain == want).all()


def test_model_equals_oracle_on_built_blocks(orc, built):
    blocks, buf, offs, lens = built
    want = orc.hash_blocks(buf, offs, lens)
    assert (K.model_hashes(buf, offs, lens) == want).all()
    for i, (n, _ph, b, _miss) in enumerate(blocks):          # pack() laid each block out unchanged
        assert b.size == n == lens[i] and orc.xxh64(b) == want[i]
    # the only rounds no word can drive onto their class: begin has no cross term, and v3 starts at 0 (nothing carries)
    unreachable = {(0, k, K.CROSS_WRAP0) for k in range(4)} | {(0, 2, K.LO_WRAP0), (0, 2, K.HI_CARRY)}
    for n, ph, _b, miss in blocks:
        assert set(miss) == {u for u in unreachable if n >= 32 and K.schedule(n, ph)[0] == u[2]}, (n, ph, miss)


def test_every_edge_class_at_every_scheduled_position(built):
    """Per lane: each of the 32 stripe positions of a chunk past the first (this includes both sides of every chunk
    boundary and of the steady-state path's 8-stripe register groups), the first round (begin) and the first step
    after it, and the last full stripe before end() -- each sees every edge class at least once, and every stripe
    lands on the class it was scheduled for."""
    blocks, buf, offs, lens = built
    _h, edges = K.model_hashes(buf, offs, lens, edges=True)
    hits = {}                                                # (position, lane) -> edge classes seen there
    for (n, ph, _b, miss), e in zip(blocks, edges):
        sched = K.schedule(n, ph)
        for s, cls in enumerate(sched):
            for k in range(4):
                assert (e[s, k] >> cls) & 1 or (s, k, cls) in miss, (n, ph, s, k, K.EDGES[cls])
        seen = [[{c for c in range(6) if (e[s, k] >> c) & 1} for k in range(4)] for s in range(len(sched))]
        for s in range(len(sched)):
            pos = [("chunk position", s % 32)] if s >= 32 else []
            pos += [("begin",)] if s == 0 else [("first step",)] if s == 1 else []
            pos += [("last stripe",)] if s == len(sched) - 1 and n >= KiB else []
            for p in pos:
                for k in range(4):
                    hits.setdefault((p, k), set()).update(seen[s][k])
    for k in range(4):
        for p in [("chunk position", i) for i in range(32)] + [("first step",), ("last stripe",)]:
            assert hits[(p, k)] == set(range(6)), (p, k, sorted(hits[(p, k)]))
        begin = set(K.BEGIN_EDGES) - ({K.LO_WRAP0, K.HI_CARRY} if K.ACC0[k] & K.M32 == 0 else set())
        assert hits[(("begin",), k)] >= begin, (k, sorted(hits[(("begin",), k)]))


@pytest.mark.parametrize("slip", sorted(K.SLIPS))
def test_slipped_round_is_caught_by_the_built_blocks(orc, built, slip):
    blocks, buf, offs, lens = built
    want = orc.hash_blocks(buf, offs, lens)
    got = K.model_hashes(buf, offs, lens, slip=K.SLIPS[slip])
    wrong = got != want
    assert all(wrong[i] for i, (n, *_rest) in enumerate(blocks) if n >= KiB), (slip, np.nonzero(~wrong)[0].tolist())


def test_slipped_rounds_agree_with_the_oracle_on_the_gpu_suites_random_blocks(orc):
    """The ring-boundary blocks of tests/test_gpu.py (about 820 000 stripes, up to 4 MiB per block): the plain 64-bit
    chain equals the oracle, and step32 -- as written and with each slip -- reproduces every one of its rounds.  So
    every slipped variant runs the same chain and computes the same hashes as the oracle: these inputs never reach
    the edges where the variants differ, nor any other edge class."""
    buf, offs, lens = ring_boundary_case()
    t_in, m, t_out, first, plain = K.plain_rounds(buf, offs, lens)
    assert (plain == orc.hash_blocks(buf, offs, lens)).all()
    lo, hi, e = K.begin32(t_in[first], m[first])
    assert ((lo | (hi << np.uint64(32))) == t_out[first]).all() and not e.any()
    rest = ~first
    tlo, thi, m, t_out = t_in[rest] & np.uint64(K.M32), t_in[rest] >> np.uint64(32), m[rest], t_out[rest]
    for slip in [0] + [K.SLIPS[s] for s in sorted(K.SLIPS)]:
        lo, hi, e = K.step32(tlo, thi, m, slip)
        assert ((lo | (hi << np.uint64(32))) == t_out).all(), slip
        assert not e.any(), (slip, [int(np.count_nonzero((e >> c) & 1)) for c in range(6)])
