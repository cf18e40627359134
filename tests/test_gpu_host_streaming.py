"""GPU tests of the host-buffer batch calls that stream their items in pieces over two streams (csrc/pieces.h): the plain
verify_each path across piece boundaries, the one rule for flat messages on every host entry point that takes them, and
the diagnostics (last_kernel_ms, last_call_ms) after each streamed call."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
OK, VERIFY, SCALARFMT, POINTDEC = 0, 1, 3, 4
INVALID_ARG = -1


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


def signed_batch(eng, n, tag):
    """n signatures by n distinct keys over messages of 1 to 53 bytes: (msgs_flat, offsets, sigs, pubkeys) as numpy arrays."""
    seeds = np.frombuffer(b"".join(hashlib.sha512(b"%s%d" % (tag, i)).digest()[:32] for i in range(n)), dtype=np.uint8).copy()
    lens = (np.arange(n) % 5) * 13 + 1
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    fl = np.random.Generator(np.random.PCG64(17)).integers(0, 256, size=int(offs[-1]), dtype=np.uint8)
    pks, sigs = eng.sign_batch_flat(seeds, fl, offs, n)
    return fl, offs, np.frombuffer(sigs, dtype=np.uint8).copy(), np.frombuffer(pks, dtype=np.uint8).copy()


def test_verify_each_plain_path_across_pieces(eng, oracle):
    """2^17 + 9 signatures by distinct keys with the per-key comb path off: three pieces on alternating streams.  A failure
    of every kind on both sides of each piece boundary is reported at exactly its index, with the oracle's kind."""
    n = (1 << 17) + 9
    fl, offs, sg, pk = signed_batch(eng, n, b"s")
    bad = [0, 65535, 65536, 131071, 131072, n - 1]
    fl[int(offs[bad[0]])] ^= 1                                            # message changed: Verify
    sg[64 * bad[1] + 63] |= 0xf0                                          # s >= l: ScalarFormat
    pk[32 * bad[2]:32 * bad[2] + 32] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)   # undecodable key
    sg[64 * bad[3]:64 * bad[3] + 32] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)   # undecodable R: Verify
    sg[64 * bad[4]] ^= 1                                                  # wrong R: Verify
    sg[64 * bad[5] + 63] |= 0xf0                                          # s >= l and an undecodable key: the key first
    pk[32 * bad[5]:32 * bad[5] + 32] = np.frombuffer((2).to_bytes(32, "little"), dtype=np.uint8)
    eng.set_option("each_comb", 0)
    try:
        for strict in (False, True):
            rc, res = eng.verify_each_flat(fl, offs, sg, pk, n, strict=strict)
            assert rc == VERIFY and [i for i, r in enumerate(res) if r] == bad, strict
            for i in bad:
                m = fl[int(offs[i]):int(offs[i + 1])].tobytes()
                assert res[i] == oracle.verify(m, sg[64 * i:64 * i + 64].tobytes(), pk[32 * i:32 * i + 32].tobytes(), strict=strict), (strict, i)
            assert [res[i] for i in bad] == [VERIFY, SCALARFMT, POINTDEC, VERIFY, VERIFY, POINTDEC]
    finally:
        eng.set_option("each_comb", 1)


def flat_callers(eng):
    """Every host entry point that takes flat messages, as f(msgs_flat, offsets, n) -> return code, for n <= 2 items
    (signatures by two keys over empty messages: valid inputs apart from the messages)."""
    from curve25519_dalek_b200.engine import _ptr as p
    lib, h = eng.lib, eng.h
    seeds = hashlib.sha512(b"flat").digest()
    empty = np.zeros(3, dtype=np.uint64)
    pks, sigs = eng.sign_batch_flat(seeds, None, empty, 2)
    _, kp, _ = eng.decompress_batch(pks, 2)
    out = (C.c_uint8 * 64)()
    res = (C.c_uint8 * 2)()
    pk_out, sig_out = (C.c_uint8 * 64)(), (C.c_uint8 * 128)()
    verdicts = (C.c_int32 * 2)()
    dst = b"QUUX-V01-CS02"
    return {
        "hash_from_bytes": lambda m, o, n: lib.dalek_b200_ristretto_hash_from_bytes_batch(h, p(m), p(o), n, out),
        "hash_to_curve": lambda m, o, n: lib.dalek_b200_edwards_hash_to_curve_batch(h, p(m), p(o), n, dst, len(dst), out),
        "encode_to_curve": lambda m, o, n: lib.dalek_b200_edwards_encode_to_curve_batch(h, p(m), p(o), n, dst, len(dst), out),
        "verify_each_flat": lambda m, o, n: lib.ed25519_b200_verify_each_flat(h, p(m), p(o), sigs, pks, n, 0, res),
        "verify_each_flat_strict": lambda m, o, n: lib.ed25519_b200_verify_each_flat(h, p(m), p(o), sigs, pks, n, 1, res),
        "verify_batch_flat": lambda m, o, n: lib.ed25519_b200_verify_batch_flat(h, p(m), p(o), sigs, pks, n),
        "verify_batch_flat_points": lambda m, o, n: lib.ed25519_b200_verify_batch_flat_points(h, p(m), p(o), sigs, pks, kp, n),
        "verify_batches_flat": lambda m, o, n: lib.ed25519_b200_verify_batches_flat(h, p(m), p(o), sigs, pks, n, 1, verdicts),
        "verify_batches_flat_points": lambda m, o, n: lib.ed25519_b200_verify_batches_flat_points(h, p(m), p(o), sigs, pks, kp, n, 1,
                                                                                                  verdicts),
        "sign_batch_flat": lambda m, o, n: lib.ed25519_b200_sign_batch_flat(h, seeds, p(m), p(o), n, pk_out, sig_out),
    }


FLAT_CALLERS = ["hash_from_bytes", "hash_to_curve", "encode_to_curve", "verify_each_flat", "verify_each_flat_strict",
                "verify_batch_flat", "verify_batch_flat_points", "verify_batches_flat", "verify_batches_flat_points",
                "sign_batch_flat"]
MSGS = np.frombuffer(b"abc\0", dtype=np.uint8).copy()
REJECTED = {
    "null_offsets": (MSGS, None),
    "first_offset_not_zero": (MSGS, np.array([1, 2, 3], dtype=np.uint64)),
    "decreasing_offsets": (MSGS, np.array([0, 2, 1], dtype=np.uint64)),
    "null_msgs_nonempty": (None, np.array([0, 1, 3], dtype=np.uint64)),
}


@pytest.mark.parametrize("case", sorted(REJECTED))
@pytest.mark.parametrize("caller", FLAT_CALLERS)
def test_flat_message_rule_rejects(eng, caller, case):
    msgs, offs = REJECTED[case]
    assert flat_callers(eng)[caller](msgs, offs, 2) == INVALID_ARG


@pytest.mark.parametrize("caller", FLAT_CALLERS)
def test_flat_message_rule_accepts(eng, caller):
    """A NULL message buffer is fine when every message is empty, and so is n = 0 with no buffers at all; a verify call may
    still return a verdict."""
    f = flat_callers(eng)[caller]
    assert f(None, np.zeros(3, dtype=np.uint64), 2) >= 0
    assert f(None, None, 0) >= 0


def test_diagnostics_report_each_streamed_call(eng):
    """After each host call that streams through the piece streamer, at 2^17 + 3 items, last_kernel_ms reports that call: a
    positive device span and one launch per piece; last_call_ms covers the span."""
    import torch
    n = (1 << 17) + 3
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.Generator(np.random.PCG64(5))
    wide = rng.integers(0, 256, size=64 * n, dtype=np.uint8)
    scal = np.ascontiguousarray(rng.integers(0, 256, size=(n, 32), dtype=np.uint8))
    scal[:, 31] &= 0x7f
    limbs, comp = eng.mul_base_batch(scal.reshape(-1), n)
    comp = np.frombuffer(comp, dtype=np.uint8).copy()
    rist = np.frombuffer(eng.ristretto_double_and_compress_batch(limbs, n), dtype=np.uint8).copy()
    offs = np.arange(n + 1, dtype=np.uint64) * 7
    msgs = rng.integers(0, 256, size=7 * n, dtype=np.uint8)
    fl, eoffs, sg, pk = signed_batch(eng, n, b"d")
    G, H = bytes(rist[:32]), bytes(rist[32:64])
    default = 3                                                         # pieces of 2^16
    calls = {
        "edwards_decompress_batch": (lambda: eng.decompress_batch(comp, n), default),
        "ristretto_decompress_batch": (lambda: eng.decompress_batch(rist, n, ristretto=True), default),
        "edwards_compress_batch": (lambda: eng.compress_batch(limbs, n), default),
        "ristretto_double_and_compress_batch": (lambda: eng.ristretto_double_and_compress_batch(limbs, n), default),
        "edwards_to_montgomery_batch": (lambda: eng.edwards_to_montgomery_batch(limbs, n), default),
        "x25519_batch": (lambda: eng.x25519_batch(scal, comp, n, want_contributory=True), default),
        "x25519_public_keys": (lambda: eng.x25519_public_keys(scal, n), default),
        "ristretto_from_uniform_bytes_batch": (lambda: eng.ristretto_from_uniform_bytes_batch(wide, n), default),
        "ristretto_hash_from_bytes_batch": (lambda: eng.ristretto_hash_from_bytes_batch(msgs, offs, n), default),
        "edwards_hash_to_curve_batch": (lambda: eng.edwards_hash_to_curve_batch(msgs, offs, n, b"dst"), default),
        "edwards_encode_to_curve_batch": (lambda: eng.edwards_encode_to_curve_batch(msgs, offs, n, b"dst"), default),
        "verify_each_flat": (lambda: eng.verify_each_flat(fl, eoffs, sg, pk, n), default),
        # comb kernel from 4096 pairs: pieces of two waves of one 384-thread CTA per SM
        "ristretto_double_base_batch": (lambda: eng.ristretto_double_base_batch(scal, scal, G, H, n), -(-n // (2 * sms * 384))),
    }
    eng.set_option("each_comb", 0)
    try:
        for name, (call, pieces) in calls.items():
            eng.compress_batch(limbs, 1)                                # one piece: a stale report would say 1 launch
            assert eng.last_kernel_ms()[1] == 1
            call()
            ms, launches = eng.last_kernel_ms()
            assert ms > 0 and launches == pieces, name
            assert eng.last_call_ms() >= ms - 1e-3, name
    finally:
        eng.set_option("each_comb", 1)
