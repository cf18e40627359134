"""CPU checks of tests/msm_digit_cases.py: its restatement of k_digits (csrc/msm.cu) is a signed-digit expansion of the
scalar, and its boundary scalars reach every edge case they are meant to, at every window width the engine accepts.
The GPU tests of tests/test_gpu_msm_variants.py rely on both."""
import random

import pytest

import msm_digit_cases as mdc
import pyref

WIDTHS = range(4, 21)


def raw_and_carries(s, c):
    """(raw bits, incoming carry) of every window, recovered from s and its digits"""
    raws, carries, carry = [], [], 0
    for w, d in enumerate(mdc.signed_digits(s, c)):
        raw = (s >> (w * c)) & ((1 << c) - 1)
        raws.append(raw)
        carries.append(carry)
        assert raw + carry - d in (0, 1 << c)         # v = d or v = d + 2^c
        carry = (raw + carry - d) >> c
    assert carry == 0                                # nothing is carried out of the last window
    return raws, carries


@pytest.mark.parametrize("c", WIDTHS)
def test_digits_expand_the_scalar(c):
    half = 1 << (c - 1)
    rnd = random.Random(c)
    scalars = mdc.boundary_scalars(c) + [rnd.getrandbits(256) for _ in range(300)] + [rnd.randrange(pyref.L) for _ in range(100)]
    for s in scalars:
        d = mdc.signed_digits(s, c)
        assert len(d) == mdc.window_count(c) == 256 // c + 1
        assert sum(x << (c * w) for w, x in enumerate(d)) == s, (c, hex(s))
        assert all(-(half - 1) <= x <= half for x in d), (c, hex(s))
        raws, carries = raw_and_carries(s, c)
        for w, x in enumerate(d):
            v = raws[w] + carries[w]
            assert x == (v - (1 << c) if v > half else v)


@pytest.mark.parametrize("c", WIDTHS)
def test_boundary_scalars_reach_every_case(c):
    half, mask = 1 << (c - 1), (1 << c) - 1
    nwin = mdc.window_count(c)
    nfull = nwin - 1
    cases = mdc.boundary_scalars(c)
    assert all(0 <= s < 2**256 for s in cases)
    assert cases == mdc.boundary_scalars(c)            # deterministic
    assert set(mdc.EDGE_SCALARS) <= set(cases)
    half_at, half_after_carry, neg_at, neg_after_carry = set(), set(), set(), set()
    zero_from_carry = chain = carry_only_last = False
    for s in cases:
        d = mdc.signed_digits(s, c)
        raws, carries = raw_and_carries(s, c)
        for w in range(nwin):
            if d[w] == half:
                half_at.add(w)
                if carries[w]:
                    half_after_carry.add(w)
            if d[w] == -(half - 1):
                neg_at.add(w)
                if carries[w]:
                    neg_after_carry.add(w)
            if d[w] == 0 and carries[w] and raws[w] == mask:
                zero_from_carry = True
        if all(carries[1:]):
            chain = True
        if raws[-1] == 0 and carries[-1] and d[-1] != 0:
            carry_only_last = True
    # +2^(c-1) (the last bucket) in every window that can hold it: all full windows, and never the last one, whose
    # top 256 mod c bits plus a carry stay below 2^(c-1)
    assert half_at == set(range(nfull))
    assert half_after_carry == set(range(1, nfull))  # window 0 never has an incoming carry
    assert neg_at == set(range(nfull))
    assert neg_after_carry == set(range(1, nfull))
    assert zero_from_carry
    assert chain
    assert carry_only_last
