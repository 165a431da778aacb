"""K1's arithmetic on the GPU (-m gpu): xxh64_blocks_kernel against the oracle on blocks built to drive its 32-bit round
onto every carry and wrap edge, on content whose words repeat, and on blocks near the 32-bit length limit.

The built blocks come from tests/_k1_chain.py; tests/test_k1_arith_host.py shows that they reach every edge class in
every lane at every stripe position, and that a round which drops one rare carry or cross term is caught by them and
missed by the random blocks the rest of the suite hashes.  Here the same kind of blocks go through both of the chain
warp's paths -- the steady state (every quad of a ring on a full, non-final 1 KiB chunk) and the per-quad slow path
(ragged or final chunks) -- in a hash_blocks launch, in a resident batch with a prior and K2, and under load from
another stream.  Every expected value comes from the oracle (oracle/xxh64_ref.c), never from a second engine run."""
import os
import threading
from pathlib import Path

import numpy as np
import pytest

import _k1_chain as K

pytestmark = pytest.mark.gpu
KiB, MiB = 1 << 10, 1 << 20
SLOT = min(max(int(os.environ.get("VMIG_SLOT_MB", "32")), 4), 1024) << 20      # the engine's staging slot
MAX_SMS = 132                             # the most SMs an H100 has: 32 quads per SM are assigned statically
# 1 KiB multiples (full last chunk), + 1..31 tail bytes, and ragged last chunks (a multiple of 32 past the last KiB)
SMALL = [KiB, 2 * KiB, 7 * KiB, 8 * KiB, KiB + 1, 3 * KiB + 17, 7 * KiB + 13, 8 * KiB + 31,
         2 * KiB + 32, 5 * KiB + 544 + 7, 8 * KiB + 992 + 31]
SEED = 0xA217


def _same_hashes(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, (what, bad[:8].tolist())


@pytest.fixture(scope="module", autouse=True)
def _gpu(vm):
    vm.init(0)
    yield
    vm.shutdown()


@pytest.fixture(scope="module")
def launch_set():
    """One hash_blocks launch of built blocks: two of 4 MiB (almost every chunk in the steady state once their ring-mates
    are done) among ~3 000 short ones at every schedule phase, shuffled, at unaligned offsets."""
    small = [b for _n, _ph, b, _miss in K.built_blocks(SMALL, SEED)]
    big = [b for _n, _ph, b, _miss in K.built_blocks([4 * MiB], SEED + 1, phases=(0, 3))]
    blocks = big + small * 45
    order = np.random.default_rng(SEED).permutation(len(blocks))
    buf, offs, lens = K.pack([blocks[i] for i in order], SEED)
    # one staging slot: the engine packs blocks at 512-byte alignment, up to 4 096 per launch
    assert len(lens) <= 4096 and sum(-(-max(int(n), 1) // 512) * 512 for n in lens) <= SLOT
    return buf, offs, lens


def test_built_blocks_through_hash_blocks(vm, orc, launch_set):
    buf, offs, lens = launch_set
    got, _ = vm.hash_blocks(buf, offs, lens)
    _same_hashes(got, orc.hash_blocks(buf, offs, lens), "built blocks")


# 9 KiB slots, all blocks 8 KiB .. 9 KiB - 1: chunks 0..6 of the statically assigned blocks run in the steady state, the
# rest (final, ragged, and blocks the work counter hands out at other times) in the slow path
RES_BB = 9 * KiB
RES_LENS = [8 * KiB, 8 * KiB + 1, 8 * KiB + 31, 8 * KiB + 32 + 5, 8 * KiB + 544, 8 * KiB + 992 + 31]
RES_N = 32 * MAX_SMS + 400


def test_built_blocks_in_a_resident_batch_with_prior(vm, orc):
    """Every slot of a batch of more than 32 x 132 blocks holds a built block, so each (ring, quad) slot of every CTA
    starts on one and the atomic work counter hands out the rest.  The prior equals the oracle's hashes with one bit
    flipped on every other block: the survivors K2 compacts are exactly those blocks."""
    distinct = [b for _n, _ph, b, _miss in K.built_blocks(RES_LENS, SEED + 2)]
    pick = [i % len(distinct) for i in range(RES_N)]
    want_distinct = np.array([orc.xxh64(b) for b in distinct], np.uint64)
    want = want_distinct[pick]
    prior = want.copy()
    flipped = np.arange(0, RES_N, 2)
    prior[flipped] ^= np.left_shift(np.uint64(1), (flipped % 64).astype(np.uint64))
    r = vm.Resident(RES_N, RES_BB)
    try:
        for i, j in enumerate(pick):
            r.upload(i, distinct[j])
        r.set_prior(prior, np.ones(RES_N, np.uint8))
        r.run(1)
        h, surv = r.results()
        _same_hashes(h, want, "resident built blocks")
        assert surv.tolist() == flipped.tolist()
    finally:
        r.close()


def _content(kind: str, n: int) -> np.ndarray:
    rng = np.random.default_rng(0xC0 + len(kind))
    if kind == "ff":
        return np.full(n, 0xFF, np.uint8)
    if kind == "80":
        return np.full(n, 0x80, np.uint8)
    if kind == "m_all_ones":                          # every word pre-multiplies to 0xFFFFFFFF_FFFFFFFF
        unit = np.frombuffer((K.M64 * K.P2_INV & K.M64).to_bytes(8, "little"), np.uint8)
    else:
        unit = rng.integers(0, 256, {"period8": 8, "period32": 32, "period1024": 1024}[kind], dtype=np.uint8)
    return np.resize(unit, n)


CONTENT = ["ff", "80", "period8", "period32", "period1024", "m_all_ones"]


def test_content_classes(vm, orc):
    """Content whose words repeat, so each lane sees one word (or one 1 KiB pattern) over and over: at 4 MiB and at a
    ragged length (a 17-stripe last chunk and a 7-byte tail)."""
    blocks = [_content(kind, n) for kind in CONTENT for n in (4 * MiB, MiB + 544 + 7)]
    buf, offs, lens = K.pack(blocks, SEED + 3)
    assert (K.M64 * K.P2_INV & K.M64) * K.P2 & K.M64 == K.M64
    got, _ = vm.hash_blocks(buf, offs, lens)
    _same_hashes(got, orc.hash_blocks(buf, offs, lens), "content classes")


def _mem_available() -> int:
    for line in Path("/proc/meminfo").read_text().splitlines():
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


NEAR_LIMIT = [(1 << 31) - 32, 1 << 31, (1 << 31) + 31, (1 << 32) - 512]
HOST_NEED = 12 << 30


def test_lengths_near_the_32_bit_limit(vm, orc):
    """One block each of 2^31 - 32, 2^31, 2^31 + 31 and 2^32 - 512 bytes (the largest block_bytes vmig_resident_open
    accepts) in one resident batch of four 2^32 - 512-byte slots: the chunk counts, descriptor lengths and the length
    term of the finish are 32-bit in the kernel.  Each block starts with a built 8 KiB + 13 prefix and goes on with the
    SplitMix64 fill; it is downloaded and hashed by the oracle."""
    if _mem_available() < HOST_NEED:
        pytest.skip(f"needs {HOST_NEED >> 30} GiB of MemAvailable to download and hash a 4 GiB block")
    bb = NEAR_LIMIT[-1]
    try:
        r = vm.Resident(len(NEAR_LIMIT), bb)
    except vm.VmigError as e:
        if e.code == vm.VMIG_ENOMEM:
            pytest.skip(f"{len(NEAR_LIMIT) * bb >> 30} GiB of HBM are not free ({e})")
        raise
    try:
        r.fill(0x5EED32)
        prefixes = [b for _n, _ph, b, _miss in K.built_blocks([8 * KiB + 13], SEED + 4, phases=range(len(NEAR_LIMIT)))]
        for i, n in enumerate(NEAR_LIMIT):
            r.upload(i, prefixes[i])
            r.set_len(i, n)
        r.set_prior(None)
        r.run(1)
        h, surv = r.results()
        assert surv.tolist() == list(range(len(NEAR_LIMIT)))
        for i, n in enumerate(NEAR_LIMIT):
            data = r.download(i, n)
            assert (data[:prefixes[i].size] == prefixes[i]).all()
            assert int(h[i]) == orc.xxh64(data), (i, n)
            del data
    finally:
        r.close()


def test_built_blocks_under_load_from_another_stream(vm, orc, launch_set):
    """The built launch once more, while a second stream keeps every SM busy with resident passes over 2.5 GiB, so the
    CTAs of the launch under test are descheduled and co-scheduled at random."""
    buf, offs, lens = launch_set
    want = orc.hash_blocks(buf, offs, lens)
    r = vm.Resident(640, 4 * MiB)
    running, stop, errs = threading.Event(), threading.Event(), []

    def load():
        try:
            r.fill(7)
            r.set_prior(None)
            while not stop.is_set():
                r.run(4)
                running.set()
        except Exception as e:      # noqa: BLE001
            errs.append(e)
        finally:
            running.set()
    t = threading.Thread(target=load)
    t.start()
    try:
        running.wait()
        got, _ = vm.hash_blocks(buf, offs, lens)
    finally:
        stop.set()
        t.join()
        r.close()
    assert not errs, errs
    _same_hashes(got, want, "built blocks under load")
