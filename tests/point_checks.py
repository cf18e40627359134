"""Checks of a returned extended point (X : Y : Z : T) -- what a caller relies on when it uses returned limbs as an
EdwardsPoint and adds to them: limbs below 2^51 and coordinates below p (canonical), Z != 0, X Y = Z T, the curve
equation in projective form, and projective equality with the expected point."""
import pyref

p, d = pyref.p, pyref.d


def coords_from_limbs(limbs):
    """20 radix-2^51 limbs (X, Y, Z, T, five each) -> four integers (not reduced)."""
    return [sum(int(limbs[5 * c + k]) << (51 * k) for k in range(5)) for c in range(4)]


def coords_from_bytes(b):
    """128 bytes X | Y | Z | T, 32 little-endian bytes each -> four integers."""
    return [int.from_bytes(b[32 * c:32 * c + 32], "little") for c in range(4)]


def affine(want):
    """(x, y) of an expected point given as a compressed Edwards encoding or as (x, y)."""
    if isinstance(want, (bytes, bytearray)):
        P = pyref.decompress(bytes(want))
        assert P is not None, bytes(want).hex()
        return P
    return want


def check_coords(coords, want, canonical=True, what=""):
    """coords: four integers.  canonical: each coordinate < p (the header's promise for returned limbs)."""
    if canonical:
        assert all(0 <= c < p for c in coords), ("coordinate >= p", what)
    X, Y, Z, T = (c % p for c in coords)
    assert Z != 0, ("Z = 0", what)
    assert X * Y % p == Z * T % p, ("T != XY/Z", what)
    assert (Y * Y - X * X) * Z * Z % p == (Z ** 4 + d * X * X * Y * Y) % p, ("not on the curve", what)
    x, y = affine(want)
    assert X == x * Z % p and Y == y * Z % p, ("not the expected point", what)


def check_limbs(limbs, want, canonical=True, what=""):
    """limbs: 20 uint64 of one point.  canonical adds: every limb < 2^51."""
    limbs = [int(v) for v in limbs]
    assert len(limbs) == 20
    if canonical:
        assert all(v < 1 << 51 for v in limbs), ("limb >= 2^51", what)
    check_coords(coords_from_limbs(limbs), want, canonical, what)


def check_limb_array(limbs, wants, canonical=True, what=""):
    """len(wants) consecutive points of 20 limbs each; wants[i] None skips point i (e.g. a rejected encoding)."""
    for i, w in enumerate(wants):
        if w is not None:
            check_limbs(limbs[20 * i:20 * i + 20], w, canonical, (what, i))
