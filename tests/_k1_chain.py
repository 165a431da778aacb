"""A CPU model of K1's XXH64 round exactly as csrc/vmig_kernels.cu computes it, and a builder of blocks that drive
that round onto its rare carry and wrap edges.

The kernel's chain (Chain::step) is not the compiler's 64-bit arithmetic.  It carries t = acc + m before the rotation,
where m = x*P2 has already been formed by the pre-multiply warp, and computes the next t = rotl(t, 31)*P1 + m' in
32-bit pieces: two funnel shifts (rl, rh), mul.lo/mul.hi of rl*P1lo, a two-IMAD cross term mhv = mh + rh*P1lo +
rl*P1hi, and an add.cc/addc pair that carries lo + ml into hi + mhv.  A slip in that lowering which only shows when a
32-bit sum wraps to an exact value fires about once in 2^32 rounds on random bytes, so random inputs do not find it.

step32() restates the step with the CUDA names and reports which edges it hit; it runs on Python ints and, unchanged,
on numpy uint64 arrays (every intermediate stays below 2^64), so model_hashes() can run the chains of many blocks at
once.  build_block() runs the four lanes forward from the seed-0 accumulators and, at each scheduled stripe, picks the
pre-multiplied word m whose step lands on the scheduled edge, then stores x = m * P2^-1 mod 2^64 (P2 is odd)."""
import random

import numpy as np

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1
P1, P2, P3, P4, P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63,
                      0x27D4EB2F165667C5)
P1lo, P1hi = P1 & M32, P1 >> 32
P2_INV = pow(P2, -1, 1 << 64)
ACC0 = ((P1 + P2) & M64, P2, 0, (-P1) & M64)          # seed 0: v1..v4, one per lane
STRIPES_PER_CHUNK = 32                                # the kernel stages 1 KiB chunks

# Edge classes: bit e of the mask step32() / begin32() return.
LO_WRAP0 = 0        # lo + ml carries and wraps to exactly 0
LO_ONES = 1         # lo + ml == 0xFFFFFFFF, no carry
HI_CARRY = 2        # a carry into hi + mhv == 0xFFFFFFFF: the high word wraps to 0
CROSS_WRAP0 = 3     # the cross-term sum mh + rh*P1lo + rl*P1hi wraps to exactly 0 (mod 2^32)
T_ZERO = 4          # t' == 0
T_ONES = 5          # t' == 2^64 - 1
EDGES = ("lo_wraps_to_0", "lo_all_ones", "carry_into_hi_all_ones", "cross_wraps_to_0", "t_zero", "t_all_ones")
BEGIN_EDGES = (LO_WRAP0, LO_ONES, HI_CARRY, T_ZERO, T_ONES)      # begin() is a plain add: it has no cross term

# Rare-edge slips a variant of step32() can carry: bit flags of its `slip` argument.
SLIP_LO_WRAP0 = 1   # the carry of lo + ml is dropped when the low sum wraps to exactly 0
SLIP_HI_CARRY = 2   # the carry into a high word of 0xFFFFFFFF is dropped
SLIP_CROSS = 4      # rl*P1hi is dropped from the cross-term sum when that sum wraps to exactly 0
SLIPS = {"lo_wrap0": SLIP_LO_WRAP0, "hi_carry": SLIP_HI_CARRY, "cross_wrap0": SLIP_CROSS}


def _mask(*flags):
    m = 0
    for e, f in enumerate(flags):
        m = m | f * (1 << e)
    return m


def begin32(acc, m):
    """Chain::begin: t = acc + m0 (the first round of a block).  Returns (tlo, thi, edges)."""
    s = (acc & M32) + (m & M32)
    carry = s >> 32
    u = (acc >> 32) + (m >> 32)
    tlo, thi = s & M32, (u + carry) & M32
    return tlo, thi, _mask(s == 1 << 32, s == M32, (carry == 1) & ((u & M32) == M32), False,
                           (tlo == 0) & (thi == 0), (tlo == M32) & (thi == M32))


def step32(tlo, thi, m, slip=0):
    """Chain::step: t' = rotl(t, 31)*P1 + m in the kernel's 32-bit pieces.  Returns (tlo', thi', edges).
    slip: SLIP_* flags of a deliberately wrong variant (0 = the kernel as written)."""
    ml, mh = m & M32, m >> 32
    rl = ((tlo << 31) | (thi >> 1)) & M32              # __funnelshift_l(thi, tlo, 31)
    rh = ((thi << 31) | (tlo >> 1)) & M32              # __funnelshift_l(tlo, thi, 31)
    p = rl * P1lo
    lo, hi = p & M32, p >> 32                          # mul.lo / mul.hi
    a = (rh * P1lo & M32) + mh                         # mad.lo a, rh, P1lo, mh   (unreduced)
    cross = (rl * P1hi & M32) + a                      # mad.lo mhv, rl, P1hi, a  (unreduced)
    mhv = cross & M32
    cross_wrap0 = (mhv == 0) & (cross != 0)
    mhv = mhv + (cross_wrap0 & ((slip & SLIP_CROSS) != 0)) * (a & M32)
    s = lo + ml                                        # add.cc
    lo_wrap0 = s == 1 << 32
    carry = (s >> 32) - (lo_wrap0 & ((slip & SLIP_LO_WRAP0) != 0))
    u = hi + mhv
    hi_carry = (carry == 1) & ((u & M32) == M32)
    carry = carry - (hi_carry & ((slip & SLIP_HI_CARRY) != 0))
    tlo, thi = s & M32, (u + carry) & M32              # addc
    return tlo, thi, _mask(lo_wrap0, s == M32, hi_carry, cross_wrap0,
                           (tlo == 0) & (thi == 0), (tlo == M32) & (thi == M32))


def end(tlo, thi):
    """Chain::end: the lane's accumulator rotl(t, 31)*P1 after its last stripe."""
    t = tlo | (thi << 32)
    return (((t << 31) | (t >> 33)) & M64) * P1 & M64


def _round(acc, x):
    t = (acc + x * P2) & M64
    return (((t << 31) | (t >> 33)) & M64) * P1 & M64


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def finish(v, tail: bytes, n: int) -> int:
    """XXH64 (seed 0) from the four lane accumulators v (or None when n < 32), the n & 31 tail bytes and the length."""
    if n >= 32:
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for x in v:
            h = ((h ^ _round(0, x)) * P1 + P4) & M64
    else:
        h = P5
    h = (h + n) & M64
    p = 0
    while p + 8 <= len(tail):
        h = (_rotl(h ^ _round(0, int.from_bytes(tail[p:p + 8], "little")), 27) * P1 + P4) & M64
        p += 8
    if p + 4 <= len(tail):
        h = (_rotl(h ^ (int.from_bytes(tail[p:p + 4], "little") * P1 & M64), 23) * P2 + P3) & M64
        p += 4
    for b in tail[p:]:
        h = (_rotl(h ^ (b * P5 & M64), 11) * P1) & M64
    h ^= h >> 33
    h = h * P2 & M64
    h ^= h >> 29
    h = h * P3 & M64
    h ^= h >> 32
    return h


class _Stripes:
    """The full stripes of a set of blocks, longest block first, back to back: row start[j] + s of m holds the four
    pre-multiplied words (m = x*P2, as the pre-multiply warp leaves them) of stripe s of block order[j]."""

    def __init__(self, buf, offs, lens):
        self.buf = np.ascontiguousarray(buf, dtype=np.uint8)
        self.offs, self.lens = [int(o) for o in offs], [int(n) for n in lens]
        self.order = sorted(range(len(self.lens)), key=lambda i: -self.lens[i])
        self.stripes = np.array([self.lens[i] // 32 for i in self.order], np.int64)
        self.start = np.concatenate([[0], np.cumsum(self.stripes)[:-1]]).astype(np.int64)
        words = [np.frombuffer(self.buf[self.offs[i]:self.offs[i] + self.lens[i] // 32 * 32].tobytes(), "<u8")
                 for i in self.order]
        self.m = np.concatenate(words + [np.empty(0, np.uint64)]).reshape(-1, 4) * np.uint64(P2)

    def rows(self):
        """(s, k, rows of stripe s): stripe s exists in the first k blocks of the order."""
        for s in range(int(self.stripes.max()) if self.stripes.size else 0):
            k = int(np.count_nonzero(self.stripes > s))
            yield s, k, self.start[:k] + s

    def hashes(self, acc):
        """XXH64 of every block from acc[j] = the four lane accumulators of block order[j]."""
        out = np.zeros(len(self.lens), np.uint64)
        for j, i in enumerate(self.order):
            o, n = self.offs[i], self.lens[i]
            out[i] = finish([int(x) for x in acc[j]] if n >= 32 else None, self.buf[o + n // 32 * 32:o + n].tobytes(), n)
        return out


def model_hashes(buf, offs, lens, slip=0, edges=False):
    """XXH64 of every block buf[offs[i]:offs[i]+lens[i]], its stripes run through begin32/step32.

    slip: one SLIP_* mask, or a list of them (one variant each; then the hashes have shape (len(slip), n)).
    edges=True also returns, per block, a uint8 array [variant, stripe, lane] of the edge masks its rounds hit.
    The chains of all blocks run side by side, one stripe at a time."""
    st = _Stripes(buf, offs, lens)
    slips = np.atleast_1d(np.asarray(slip, dtype=np.uint64))
    nv, nb = slips.size, len(st.lens)
    sl = slips.reshape(nv, 1, 1)
    tlo = np.zeros((nv, nb, 4), np.uint64)
    thi = np.zeros((nv, nb, 4), np.uint64)
    rec = np.zeros((nv, st.m.shape[0], 4), np.uint8) if edges else None
    for s, k, rows in st.rows():
        ms = st.m[rows]
        if s == 0:
            lo, hi, e = begin32(np.broadcast_to(np.array(ACC0, np.uint64), (nv, k, 4)), np.broadcast_to(ms, (nv, k, 4)))
        else:
            lo, hi, e = step32(tlo[:, :k], thi[:, :k], ms, sl)
        tlo[:, :k], thi[:, :k] = lo, hi
        if edges:
            rec[:, rows] = e
    acc = end(tlo, thi)
    out = np.stack([st.hashes(acc[v]) for v in range(nv)])
    out = out if np.ndim(slip) else out[0]
    if not edges:
        return out
    per_block = [None] * nb
    for j, i in enumerate(st.order):
        r = rec[:, st.start[j]:st.start[j] + st.stripes[j]]
        per_block[i] = r if np.ndim(slip) else r[0]
    return out, per_block


def plain_rounds(buf, offs, lens):
    """Every round of every block, by the compiler's 64-bit arithmetic instead of the 32-bit pieces: arrays with one
    row per stripe (all blocks back to back) and one column per lane -- t_in (the carried state a step starts from;
    the accumulator for a block's first stripe), m (its pre-multiplied word), t_out (the state after it) and first
    (the row is a block's first stripe) -- and the XXH64 of every block.  It costs a few numpy operations per stripe,
    so step32 can then be checked on every round of long random blocks at once."""
    st = _Stripes(buf, offs, lens)
    t_in, t_out = np.zeros_like(st.m), np.zeros_like(st.m)
    first = np.zeros(st.m.shape[0], bool)
    t = np.zeros((len(st.lens), 4), np.uint64)
    for s, k, rows in st.rows():
        if s == 0:
            first[rows] = True
            t_in[rows] = np.array(ACC0, np.uint64)
            t[:k] = t_in[rows] + st.m[rows]
        else:
            t_in[rows] = t[:k]
            t[:k] = ((t[:k] << np.uint64(31)) | (t[:k] >> np.uint64(33))) * np.uint64(P1) + st.m[rows]
        t_out[rows] = t[:k]
    return t_in, st.m, t_out, first, st.hashes(end(t & M32, t >> np.uint64(32)))


# ------------------------------------------------------------------------------------------ the builder
def schedule(length: int, phase: int):
    """The edge class of every stripe: (phase + position in the chunk + chunk index) mod 6.  Within six chunks every
    position of a chunk meets every class; across the six phases so do the first round and the last full stripe."""
    return [(phase + s % STRIPES_PER_CHUNK + s // STRIPES_PER_CHUNK) % len(EDGES) for s in range(length // 32)]


def _odd_below(n, rnd):
    """A random odd number below n (0 when n == 1).  A carry into a high word of all ones leaves t = {odd, 0}, so the
    next step's rl = (tlo << 31) | (thi >> 1) is not 0 and can carry again."""
    return 2 * rnd.randrange(n // 2) + 1 if n > 1 else 0


def _m_begin(acc, e, rnd):
    """The m0 whose begin(acc, m0) lands on edge e, or None where no m0 can (acc's low word is 0: nothing carries)."""
    alo, ahi = acc & M32, acc >> 32
    if e == LO_WRAP0:
        return None if alo == 0 else ((-alo) & M32) | rnd.getrandbits(32) << 32
    if e == LO_ONES:
        return (M32 - alo) | rnd.getrandbits(32) << 32
    if e == HI_CARRY:
        return None if alo == 0 else ((1 << 32) - alo + _odd_below(alo, rnd)) | ((M32 - ahi) & M32) << 32
    if e == T_ZERO:
        return (-acc) & M64
    if e == T_ONES:
        return (M64 - acc) & M64
    return None                                                   # CROSS_WRAP0: begin has no cross term


def _m_step(t, e, rnd):
    """The m whose step from carried state t lands on edge e, or None where no m can."""
    r = ((t << 31) | (t >> 33)) & M64
    rp = r * P1 & M64                                             # = {lo, hi + cross} of the kernel's pieces
    lo, hi = rp & M32, rp >> 32
    if e == LO_WRAP0:
        return None if lo == 0 else ((-lo) & M32) | rnd.getrandbits(32) << 32
    if e == LO_ONES:
        return (M32 - lo) | rnd.getrandbits(32) << 32
    if e == HI_CARRY:
        return None if lo == 0 else ((1 << 32) - lo + _odd_below(lo, rnd)) | ((M32 - hi) & M32) << 32
    if e == CROSS_WRAP0:
        rl, rh = r & M32, r >> 32
        c = (rh * P1lo & M32) + (rl * P1hi & M32)
        return None if c == 0 else rnd.getrandbits(32) | ((-c) & M32) << 32
    if e == T_ZERO:
        return (-rp) & M64
    return (M64 - rp) & M64                                       # T_ONES


def build_block(length: int, sched, seed: int):
    """`length` bytes whose stripes land, in every lane, on the edge class sched[s] (None: a random word).  The tail
    after the last full stripe is random.  Returns (uint8 array, misses): misses lists the (stripe, lane, class) that no
    word can reach from the state the lane is in -- with schedule(), only begin's carries in lane 2 (v3), whose
    accumulator starts at 0."""
    rnd = random.Random(seed)
    n = length // 32
    assert len(sched) == n, (len(sched), n)
    xs, misses = [0] * (4 * n), []
    for k in range(4):
        t = 0
        for s in range(n):
            e = sched[s]
            m = None if e is None else (_m_begin(ACC0[k], e, rnd) if s == 0 else _m_step(t, e, rnd))
            if m is None:
                if e is not None:
                    misses.append((s, k, e))
                m = rnd.getrandbits(64) * P2 & M64
            xs[4 * s + k] = m * P2_INV & M64
            if s == 0:
                t = (ACC0[k] + m) & M64
            else:
                r = ((t << 31) | (t >> 33)) & M64
                t = (r * P1 + m) & M64
    tail = bytes(rnd.getrandbits(8) for _ in range(length % 32))
    out = np.frombuffer(np.array(xs, "<u8").tobytes() + tail, np.uint8)
    return out, misses


def built_blocks(lengths, seed: int, phases=range(6)):
    """Every length built at every schedule phase: [(length, phase, bytes, misses)]."""
    out = []
    for i, n in enumerate(lengths):
        for ph in phases:
            b, miss = build_block(n, schedule(n, ph), seed * 1_000_003 + i * 101 + ph)
            out.append((n, ph, b, miss))
    return out


def pack(blocks, seed: int):
    """Lay blocks out in one buffer at unaligned offsets (gaps of 1..17 random bytes): (buf, offs, lens)."""
    rng = np.random.default_rng(seed)
    lens = np.array([b.size for b in blocks], np.uint32)
    gaps = rng.integers(1, 18, len(blocks)).astype(np.uint64)
    offs = np.cumsum(gaps + np.concatenate([[0], lens[:-1]]).astype(np.uint64)).astype(np.uint64)
    buf = rng.integers(0, 256, int(offs[-1]) + int(lens[-1]) + 8, dtype=np.uint8)
    for o, b in zip(offs, blocks):
        buf[int(o):int(o) + b.size] = b
    return buf, offs, lens
