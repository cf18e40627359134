"""Signed radix-2^c digits of the bucket MSM and scalars that reach their edge cases (test input synthesis).

k_digits (csrc/msm.cu) cuts a 256-bit scalar into nwin = 256 // c + 1 windows of c bits.  Window w adds the carry of
window w - 1 to its raw bits; a value v > 2^(c-1) becomes the digit v - 2^c and carries one into window w + 1.  Digits
therefore lie in [-(2^(c-1) - 1), 2^(c-1)], and digit +-d lands in bucket d - 1 of its window, so +2^(c-1) is the only
digit that reaches the last bucket.  The 256 // c full windows hold the scalar; the last window holds its top
256 mod c bits (none when c divides 256) plus the carry out of the full windows."""
import pyref

EDGE_SCALARS = (0, 1, pyref.L - 1, pyref.L, 2**252, 2**255 - 1, 2**255, 2**256 - 1)


def window_count(c):
    return 256 // c + 1


def signed_digits(s, c):
    """The digits k_digits gives the scalar s (0 <= s < 2^256) at width c, window 0 first."""
    assert 0 <= s < 2**256 and 4 <= c <= 20
    mask, half = (1 << c) - 1, 1 << (c - 1)
    digits, carry = [], 0
    for w in range(window_count(c)):
        v = ((s >> (w * c)) & mask) + carry
        if v > half:
            digits.append(v - (1 << c))
            carry = 1
        else:
            digits.append(v)
            carry = 0
    return digits


def boundary_scalars(c):
    """Deterministic scalars whose digits at width c reach the edges of k_digits:
    - +2^(c-1) in every full window, with and without an incoming carry;
    - -(2^(c-1) - 1), with and without an incoming carry;
    - zero digits made by a carry (raw = 2^c - 1 plus the carry);
    - a carry out of every window but the last, and a non-zero last digit made by that carry alone;
    - the edge values EDGE_SCALARS."""
    nfull = 256 // c
    mask, half = (1 << c) - 1, 1 << (c - 1)

    def windows(f):                                  # f(w) = raw bits of full window w
        return sum(f(w) << (c * w) for w in range(nfull))

    out = [
        windows(lambda w: half),                                   # +half everywhere, no carry
        windows(lambda w: mask if w % 2 == 0 else half - 1),       # -1 carries into half - 1: +half in odd windows
        windows(lambda w: mask if w % 2 == 1 else half - 1),       # ... and in even windows
        windows(lambda w: half + 1 if w % 2 == 0 else 0),          # -(half - 1) in even windows, +1 after it
        windows(lambda w: half + 1 if w % 2 == 1 else 0),          # ... in odd windows
        windows(lambda w: half + 1 if w == 0 else half),           # half + carry: -(half - 1) and a carry in every window
        windows(lambda w: mask),                                   # -1, then raw 2^c - 1 + carry = 0 up to the last window
    ]
    for w in range(nfull):                                         # each boundary digit alone in one window
        out.append(half << (c * w))
        out.append((half + 1) << (c * w))
    out += EDGE_SCALARS
    return out
