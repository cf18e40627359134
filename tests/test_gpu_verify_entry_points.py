"""GPU tests of the argument rules of every Ed25519 verify entry point (the nine verify_batch[es] calls and the three
per-signature ones), and of the per-call transcript length of verify_batches, which must not outlive the call."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
OK, INVALID_ARG = 0, -1
N = 4


@pytest.fixture(scope="module")
def eng():
    import curve25519_dalek_b200 as pkg
    e = pkg.Engine(0)
    yield e
    e.close()


def signed(eng, n, tag, nkeys=None):
    """n valid signatures over 1- to 53-byte messages by `nkeys` keys (default: all distinct):
    (msgs_flat, offsets, sigs, pubkeys, seeds) as numpy arrays."""
    nkeys = nkeys or n
    seeds_k = np.frombuffer(b"".join(hashlib.sha512(b"%s%d" % (tag, k)).digest()[:32] for k in range(nkeys)), dtype=np.uint8)
    seeds = np.ascontiguousarray(seeds_k.reshape(nkeys, 32)[np.arange(n) % nkeys])
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum((np.arange(n) % 5) * 13 + 1)
    fl = np.random.Generator(np.random.PCG64(5)).integers(0, 256, size=int(offs[-1]), dtype=np.uint8)
    pks, sigs = eng.sign_batch_flat(seeds, fl, offs, n)
    return fl, offs, np.frombuffer(sigs, dtype=np.uint8).copy(), np.frombuffer(pks, dtype=np.uint8).copy(), seeds


@pytest.fixture(scope="module")
def bufs(eng):
    """Valid inputs for N signatures, in host memory ("h") and device memory ("d"), with an output buffer for every
    kind of call; a case sets one of them to None."""
    import torch
    fl, offs, sg, pk, seeds = signed(eng, N, b"args")
    rc, limbs, ok = eng.decompress_batch(pk.tobytes(), N)
    assert rc == 0 and all(ok)
    kp = np.frombuffer(limbs, dtype=np.uint64).copy()
    phs = np.frombuffer(b"".join(hashlib.sha512(b"ph%d" % i).digest() for i in range(N)), dtype=np.uint8).copy()
    rc, ph_sigs = eng.sign_prehashed(seeds, N, phs, N)
    assert rc == OK
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(v if v.dtype == np.uint8 else v.view(np.int64)).to(dev) for k, v in
         (("msgs", fl), ("offs", offs), ("sigs", sg), ("keys", pk), ("kp", kp))}
    torch.cuda.synchronize()
    msg_bufs = [C.create_string_buffer(fl[int(offs[i]):int(offs[i + 1])].tobytes()) for i in range(N)]
    return {
        "h": {"msgs": fl, "offs": offs, "sigs": sg, "keys": pk, "kp": kp},
        "d": {k: v.data_ptr() for k, v in d.items()}, "d_tensors": d,
        "ptrs": {"msgs": (C.c_void_p * N)(*[C.addressof(b) for b in msg_bufs]),
                 "offs": (C.c_size_t * N)(*[int(offs[i + 1] - offs[i]) for i in range(N)]), "sigs": sg, "keys": pk},
        "msg_bufs": msg_bufs,
        "ph": {"msgs": phs, "sigs": np.frombuffer(ph_sigs, dtype=np.uint8).copy(), "keys": pk},
    }


def _p(x):
    from curve25519_dalek_b200.engine import _ptr
    return _ptr(x)


# entry point -> (input set, the buffers it requires when n > 0, call(lib, h, b, n, batch_size) -> return code).
# b maps msgs / offs / sigs / keys / kp / out to a buffer or None (for verify_batch msgs / offs are the array of message
# pointers and the array of lengths).  Null message offsets of the host calls are
# covered by test_gpu_host_streaming.py, the null prehash and the context of verify_prehashed_each by test_gpu_sign.py.
ENTRY = {
    "verify_batch": ("ptrs", ("msgs", "offs", "sigs", "keys"),
                     lambda L, h, b, n, bs: L.ed25519_b200_verify_batch(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]), _p(b["keys"]), n)),
    "verify_batch_flat": ("h", ("sigs", "keys"),
                          lambda L, h, b, n, bs: L.ed25519_b200_verify_batch_flat(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]),
                                                                                  _p(b["keys"]), n)),
    "verify_batch_flat_dev": ("d", ("offs", "sigs", "keys"),
                              lambda L, h, b, n, bs: L.ed25519_b200_verify_batch_flat_dev(h, b["msgs"], b["offs"], b["sigs"], b["keys"], n,
                                                                                          0)),
    "verify_batch_flat_points": ("h", ("sigs", "keys", "kp"),
                                 lambda L, h, b, n, bs: L.ed25519_b200_verify_batch_flat_points(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]),
                                                                                                _p(b["keys"]), _p(b["kp"]), n)),
    "verify_batch_flat_points_dev": ("d", ("offs", "sigs", "keys", "kp"),
                                     lambda L, h, b, n, bs: L.ed25519_b200_verify_batch_flat_points_dev(h, b["msgs"], b["offs"], b["sigs"],
                                                                                                        b["keys"], b["kp"], n)),
    "verify_batches_flat": ("h", ("sigs", "keys", "out"),
                            lambda L, h, b, n, bs: L.ed25519_b200_verify_batches_flat(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]),
                                                                                      _p(b["keys"]), n, bs, _p(b["out"]))),
    "verify_batches_flat_dev": ("d", ("offs", "sigs", "keys", "out"),
                                lambda L, h, b, n, bs: L.ed25519_b200_verify_batches_flat_dev(h, b["msgs"], b["offs"], b["sigs"], b["keys"], n,
                                                                                              bs, _p(b["out"]))),
    "verify_batches_flat_points": ("h", ("sigs", "keys", "kp", "out"),
                                   lambda L, h, b, n, bs: L.ed25519_b200_verify_batches_flat_points(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]),
                                                                                                    _p(b["keys"]), _p(b["kp"]), n, bs,
                                                                                                    _p(b["out"]))),
    "verify_batches_flat_points_dev": ("d", ("offs", "sigs", "keys", "kp", "out"),
                                       lambda L, h, b, n, bs: L.ed25519_b200_verify_batches_flat_points_dev(h, b["msgs"], b["offs"], b["sigs"],
                                                                                                            b["keys"], b["kp"], n, bs,
                                                                                                            _p(b["out"]))),
    "verify_each_flat": ("h", ("sigs", "keys", "out"),
                         lambda L, h, b, n, bs: L.ed25519_b200_verify_each_flat(h, _p(b["msgs"]), _p(b["offs"]), _p(b["sigs"]), _p(b["keys"]),
                                                                                n, 0, _p(b["out"]))),
    "verify_each_flat_dev": ("d", ("offs", "sigs", "keys", "out"),
                             lambda L, h, b, n, bs: L.ed25519_b200_verify_each_flat_dev(h, b["msgs"], b["offs"], b["sigs"], b["keys"], n, 0,
                                                                                        _p(b["out"]))),
    "verify_prehashed_each": ("ph", ("sigs", "keys", "out"),
                              lambda L, h, b, n, bs: L.ed25519_b200_verify_prehashed_each(h, _p(b["msgs"]), None, 0, _p(b["sigs"]),
                                                                                          _p(b["keys"]), n, 0, _p(b["out"]))),
}
BATCHES = [e for e in ENTRY if e.startswith("verify_batches")]

# (entry, case, n, batch_size, buffer set to None or "all", expected return code)
CASES = [(e, "valid", N, 2, None, OK) for e in ENTRY]
CASES += [(e, "n0_all_null", 0, 1, "all", OK) for e in ENTRY]
CASES += [(e, "null_" + r, N, 2, r, INVALID_ARG) for e in ENTRY for r in ENTRY[e][1]]
CASES += [(e, "batch_size_%d" % bs, n, bs, nul, INVALID_ARG) for e in BATCHES
          for bs in (0, (1 << 20) + 1) for n, nul in ((N, None), (0, "all"))]
CASES += [(e, "batch_size_2^20", N, 1 << 20, None, OK) for e in BATCHES]


def call_case(eng, bufs, entry, n, bs, nul):
    kind, _, fn = ENTRY[entry]
    out = (C.c_int32 * N)() if entry in BATCHES else (C.c_uint8 * N)()
    b = dict(bufs[kind], out=out)
    for k in b:
        if nul == "all" or k == nul:
            b[k] = None
    return fn(eng.lib, eng.h, b, n, bs)


@pytest.mark.parametrize("entry,case,n,bs,nul,want", CASES, ids=["%s-%s" % (c[0], c[1]) + ("-n0" if c[2] == 0 and c[1] != "n0_all_null" else "")
                                                                for c in CASES])
def test_verify_entry_point_arguments(eng, bufs, entry, case, n, bs, nul, want):
    assert call_case(eng, bufs, entry, n, bs, nul) == want


def test_rejected_calls_leave_last_call_ms(eng, bufs):
    """A call rejected for its arguments enqueues nothing and leaves the device time of the last call as it was."""
    assert call_case(eng, bufs, "verify_batch_flat", N, 0, None) == OK
    ms = eng.last_call_ms()
    for entry, _, n, bs, nul, want in CASES:
        if want == INVALID_ARG:
            assert call_case(eng, bufs, entry, n, bs, nul) == INVALID_ARG
            assert eng.last_call_ms() == ms, (entry, nul, bs)


@pytest.mark.parametrize("device", [False, True])
def test_verify_chunk_survives_verify_batches(eng, oracle, device):
    """verify_batches runs one transcript per batch without touching the user's verify_chunk: a verify_batch call after
    it still draws the z_i of 64-signature transcripts."""
    import torch
    n = 300
    fl, offs, sg, pk, _ = signed(eng, n, b"chunk", nkeys=7)
    msgs = [fl[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]
    sigs = [sg[64 * i:64 * i + 64].tobytes() for i in range(n)]
    pks = [pk[32 * i:32 * i + 32].tobytes() for i in range(n)]
    rc_o, zs_o = oracle.verify_batch(msgs, sigs, pks, chunk=64, want_zs=True)
    assert rc_o == OK
    if device:
        dev = torch.device("cuda", 0)
        t = [torch.from_numpy(x if x.dtype == np.uint8 else x.view(np.int64)).to(dev) for x in (fl, offs, sg, pk)]
        args = [x.data_ptr() for x in t]
    else:
        args = [fl, offs, sg, pk]
    eng.set_option("verify_chunk", 64)
    try:
        rc, v = eng.verify_batches_flat(*args, n, 32, device_ptrs=device)
        assert rc == OK and v == [OK] * ((n + 31) // 32)
        assert eng.verify_batch_flat(*args, n, device_ptrs=device) == OK
        assert eng.last_zs(n) == zs_o
    finally:
        eng.set_option("verify_chunk", 0)
