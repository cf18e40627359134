"""MSM inputs over a pool of oracle points whose sums have an exact and cheap reference (test input synthesis).

Pool entry j is the point t_j B + m_j T8, T8 the order-8 point of torsion_cases: NPOOL entries with m_j = 0, the first
NSHIFT of them again shifted by T8 (m_j = 1), and the eight points k T8 of E[8] (t_j = 0, m_j = k; k = 0 is the identity).
Then for any scalars below 2^256

    sum s_i P_{idx_i} = ((sum s_i t_{idx_i}) mod l) B + ((sum s_i m_{idx_i}) mod 8) T8,

so the expected value of an MSM of any size costs one pass of Python integer arithmetic and two oracle multiplications."""
import random

import numpy as np

import pyref
import torsion_cases

L, P = pyref.L, pyref.p
NPOOL, NSHIFT = 64, 8
SHIFTED = NPOOL                  # entries SHIFTED + k: entry k + T8
E8 = NPOOL + NSHIFT              # entries E8 + k: k T8, k = 0 .. 7
MASK51 = np.uint64((1 << 51) - 1)


def b32(x):
    return x.to_bytes(32, "little")


def scalar_array(values):
    """Python integers below 2^256 -> (n, 32) uint8, little-endian rows"""
    return np.frombuffer(b"".join(b32(v) for v in values), dtype=np.uint8).reshape(-1, 32).copy()


def scalar_ints(arr):
    """(n, 32) uint8 -> Python integers"""
    b = np.ascontiguousarray(arr).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def limbs51(coord_bytes):
    """(n, 4, 32) uint8 coordinates below 2^255, little-endian -> (n, 20) uint64 radix-2^51 limbs"""
    n = coord_bytes.shape[0]
    w = np.ascontiguousarray(coord_bytes).view("<u8").reshape(n, 4, 4)
    out = np.empty((n, 4, 5), dtype=np.uint64)
    for k in range(5):
        i, off = divmod(51 * k, 64)
        v = w[:, :, i] >> np.uint64(off)
        if off + 51 > 64:
            v |= w[:, :, i + 1] << np.uint64(64 - off)
        out[:, :, k] = v & MASK51
    return out.reshape(n, 20)


def coords(limbs):
    """20 radix-2^51 limbs -> (X, Y, Z, T) as integers mod p"""
    return [sum(int(limbs[5 * c + k]) << (51 * k) for k in range(5)) % P for c in range(4)]


def rescaled(xyzt_list, rnd):
    """(n, 20) limbs of the extended points (lambda_i X : lambda_i Y : lambda_i Z : lambda_i T), each with its own
    lambda_i != 0, 1 drawn from rnd"""
    out = bytearray()
    for xyzt in xyzt_list:
        lam = rnd.randrange(2, P)
        for v in xyzt:
            out += b32(v * lam % P)
    return limbs51(np.frombuffer(bytes(out), dtype=np.uint8).reshape(-1, 4, 32))


class Pool:
    def __init__(self, oracle, seed=0x9001):
        self.oracle = oracle
        rnd = random.Random(seed)
        self.B = oracle.basepoint()
        self.T8 = oracle.decompress(torsion_cases.T8)
        tors = [oracle.identity()] + torsion_cases.torsion_points(oracle)
        t = [rnd.randrange(1, L) for _ in range(NPOOL)]
        base = [oracle.scalarmul(b32(x), self.B) for x in t]
        self.t = t + t[:NSHIFT] + [0] * 8
        self.m = [0] * NPOOL + [1] * NSHIFT + list(range(8))
        self.points = base + [oracle.add(p, self.T8) for p in base[:NSHIFT]] + tors
        self.size = len(self.points)
        self.comp = np.frombuffer(b"".join(oracle.compress(p) for p in self.points), dtype=np.uint8).reshape(-1, 32).copy()
        self.xyzt = [coords(oracle.p3_limbs(p)) for p in self.points]

    def random_indices(self, rng, n, shifted=8):
        """n pool indices: entries without torsion, and about one in `shifted` replaced by a T8-shifted entry"""
        idx = rng.integers(0, NPOOL, size=n)
        sh = rng.random(n) < 1.0 / shifted
        idx[sh] = SHIFTED + rng.integers(0, NSHIFT, size=int(sh.sum()))
        return idx

    def sums(self, scalars, idx):
        """(sum s_i t_i mod l, sum s_i m_i mod 8) of Python-integer scalars over pool indices"""
        k = m = 0
        t, mm = self.t, self.m
        for s, j in zip(scalars, idx.tolist() if hasattr(idx, "tolist") else idx):
            k += s * t[j]
            if mm[j]:
                m += s * mm[j]
        return k % L, m % 8

    def encode(self, k, m=0):
        """the compressed encoding of (k mod l) B + (m mod 8) T8"""
        r = self.oracle.scalarmul(b32(k % L), self.B)
        if m % 8:
            r = self.oracle.add(r, self.oracle.scalarmul(b32(m % 8), self.T8))
        return self.oracle.compress(r)

    def want(self, scalars, idx):
        return self.encode(*self.sums(scalars, idx))

    def extended(self, idx, rnd):
        """(n, 20) uint64: pool entries idx, every point rescaled by its own lambda"""
        return rescaled([self.xyzt[j] for j in idx.tolist()], rnd)
