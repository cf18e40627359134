"""Several engine contexts at once, interleaved calls on one context, and errors that must not leak into later calls.

include/dalek_b200.h promises that different contexts may be used concurrently, one thread each.  Kernel attributes
such as the dynamic shared-memory limit belong to the kernel on the device, so every context shares them; workspaces
belong to one context and are regrown by whichever entry point needs more.  These tests run contexts side by side with
different sizes, entry points and options, and check every result against a value computed before any thread starts:
the CPU oracle, or the identity  sum s_i [k_i]B = [sum s_i k_i mod l]B, exact at any n.  No check compares one
engine's output with another's."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import pyref

pytestmark = pytest.mark.gpu

L = pyref.L
BARRIER_S = 120                      # a thread that never reaches the barrier fails the test instead of hanging it
JOIN_S = 300


# ---- inputs with known results ------------------------------------------------------------------------------------
class Pool:
    """m points P_j = [k_j]B: 32-byte encodings, and extended limbs with Z != 1 (3P - 2P)."""

    def __init__(self, oracle, m=64, seed=1):
        rnd = random.Random(seed)
        self.oracle = oracle
        B = oracle.basepoint()
        self.k = [rnd.randrange(1, L) for _ in range(m)]
        pts = [oracle.scalarmul(k.to_bytes(32, "little"), B) for k in self.k]
        self.enc = np.frombuffer(b"".join(oracle.compress(p) for p in pts), dtype=np.uint8).reshape(m, 32)
        self.ext = np.array([oracle.p3_limbs(oracle.sub(oracle.add(oracle.double(p), p), oracle.double(p))) for p in pts],
                            dtype=np.uint64)

    def times_base(self, k):
        return self.oracle.compress(self.oracle.scalarmul((k % L).to_bytes(32, "little"), self.oracle.basepoint()))


class MsmCase:
    """n scalars (bit 255 clear) and n points drawn from a pool; `want` is the CompressedEdwardsY of the MSM."""

    def __init__(self, pool, n, seed):
        rng = np.random.default_rng(seed)
        sc = rng.integers(0, 256, size=(max(n, 1), 32), dtype=np.uint8)[:n]
        sc[:, 31] &= 0x7F
        if n >= 4:
            sc[0] = 0                                   # a zero scalar, l - 1 and 2^255 - 1
            sc[1] = np.frombuffer((L - 1).to_bytes(32, "little"), dtype=np.uint8)
            sc[2] = np.frombuffer((2**255 - 1).to_bytes(32, "little"), dtype=np.uint8)
        self.idx = rng.integers(0, len(pool.k), size=n)
        self.n = n
        self.sb = sc.tobytes()
        self.comp = pool.enc[self.idx].tobytes()
        self.ext = pool.ext[self.idx].copy()
        self.ints = [int.from_bytes(self.sb[32 * i:32 * i + 32], "little") for i in range(n)]
        self.pool = pool
        self.want = self.segment_want(0, n)

    def segment_want(self, lo, hi):
        acc = [0] * len(self.pool.k)
        for i in range(lo, hi):
            acc[self.idx[i]] += self.ints[i]
        return self.pool.times_base(sum(a * k for a, k in zip(acc, self.pool.k)))

    def points(self, fmt):
        return self.comp if fmt == 0 else self.ext


def on_device(*bufs):
    import torch
    out = []
    for b in bufs:
        a = np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray)) else b.view(np.uint8).reshape(-1)
        out.append(torch.from_numpy(a.copy()).to("cuda:0"))
    return out


class SigCase:
    """n Ed25519 signatures over distinct messages by `keys` keys (oracle-signed), and a copy with message `bad` altered."""

    def __init__(self, oracle, n, keys, seed, bad):
        rnd = random.Random(seed)
        seeds = [rnd.randbytes(32) for _ in range(keys)]
        pks = [oracle.public_key(s) for s in seeds]
        self.msgs = [rnd.randbytes(rnd.randrange(0, 80)) for _ in range(n)]
        self.sigs = b"".join(oracle.sign(m, seeds[i % keys]) for i, m in enumerate(self.msgs))
        self.pks = b"".join(pks[i % keys] for i in range(n))
        self.n, self.bad = n, bad
        self.offs = np.zeros(n + 1, dtype=np.uint64)
        self.offs[1:] = np.cumsum([len(m) for m in self.msgs])
        self.flat = np.frombuffer(b"".join(self.msgs) + b"\0", dtype=np.uint8).copy()
        self.flat_bad = self.flat.copy()
        if len(self.msgs[bad]) == 0:
            raise ValueError("the altered message must not be empty")
        self.flat_bad[int(self.offs[bad])] ^= 1
        bad_msgs = list(self.msgs)
        bad_msgs[bad] = bytes(self.flat_bad[int(self.offs[bad]):int(self.offs[bad + 1])])
        self.bad_msgs = bad_msgs
        sig_list, pk_list = [self.sigs[64 * i:64 * i + 64] for i in range(n)], [self.pks[32 * i:32 * i + 32] for i in range(n)]
        self.want_bad = oracle.verify_batch(bad_msgs, sig_list, pk_list)
        self.want_batches = {}
        for size in (256,):
            self.want_batches[size] = [oracle.verify_batch(bad_msgs[k:k + size], sig_list[k:k + size], pk_list[k:k + size])
                                       if k <= bad < k + size else 0 for k in range(0, n, size)]


def last_error(eng):
    return eng.lib.dalek_b200_last_error(eng.h).decode(errors="replace")


def run_threads(jobs, rounds):
    """jobs: (name, engine, [(label, fn(engine))]).  Every thread waits at one barrier, then runs its steps `rounds`
    times.  A step fails by raising; the failures are reported after the join with thread, round, call and last_error."""
    barrier = threading.Barrier(len(jobs), timeout=BARRIER_S)
    failures, lock = [], threading.Lock()

    def worker(name, eng, steps):
        try:
            barrier.wait()
        except threading.BrokenBarrierError:
            with lock:
                failures.append("%s: the barrier broke" % name)
            return
        for r in range(rounds):
            for i, (label, fn) in enumerate(steps):
                try:
                    fn(eng)
                except Exception as exc:                    # noqa: BLE001 -- reported below, with the engine's last error
                    with lock:
                        failures.append("%s round %d call %d (%s): %r; last_error=%r" % (name, r, i, label, exc, last_error(eng)))

    threads = [threading.Thread(target=worker, args=job, name=job[0]) for job in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_S)
    assert not any(t.is_alive() for t in threads), "a thread did not finish"
    assert not failures, "\n".join(failures)


# ---- steps: one engine call and its check ---------------------------------------------------------------------------
def msm_step(case, fmt=0, device=None, options=()):
    def step(eng):
        for name, v in options:
            eng.set_option(name, v)
        try:
            if device is not None:
                rc, got, _ = eng.edwards_vartime_msm(device[0], device[1], case.n, point_fmt=fmt, device_ptrs=True)
            else:
                rc, got, _ = eng.edwards_vartime_msm(case.sb, case.points(fmt), case.n, point_fmt=fmt)
        finally:
            for name, _ in options:
                eng.set_option(name, DEFAULTS[name])
        assert rc == 0 and got == case.want, (case.n, fmt, rc)
    return step


DEFAULTS = {"window_bits": 0, "small_straus": 1, "host_chunks": 8, "precomp_tables": 0}


def verify_batch_step(sc, bad=False):
    def step(eng):
        rc = eng.verify_batch_flat(sc.flat_bad if bad else sc.flat, sc.offs, sc.sigs, sc.pks, sc.n)
        assert rc == (sc.want_bad if bad else 0), rc
    return step


def verify_batches_step(sc, batch, want):
    def step(eng):
        rc, verdicts = eng.verify_batches_flat(sc.flat_bad, sc.offs, sc.sigs, sc.pks, sc.n, batch)
        assert rc == 1 and verdicts == want and 1 in want, verdicts
    return step


def msm_batch_step(case, offsets, fmt=0, constant_time=False):
    offs = np.array(offsets, dtype=np.uint64)
    want = b"".join(case.segment_want(a, b) for a, b in zip(offsets[:-1], offsets[1:]))
    m = len(offsets) - 1

    def step(eng):
        rc, got, ok, _ = eng.msm_batch(case.sb, case.points(fmt), offs, m, point_fmt=fmt, constant_time=constant_time)
        assert rc == 0 and ok == b"\x01" * m and got == want, rc
    return step


def partial_combine_step(case, ranks=2):
    from curve25519_dalek_b200.sharding import shard_range, shard_size
    n_shard = shard_size(case.n, ranks)

    def step(eng):
        nwin = eng.msm_window_count(n_shard)
        allw = (C.c_uint64 * (20 * nwin * ranks))()
        for r in range(ranks):
            lo, hi = shard_range(case.n, r, ranks)
            rc, w = eng.edwards_msm_partial(case.sb[32 * lo:32 * hi], case.comp[32 * lo:32 * hi], hi - lo, n_shard)
            assert rc == 0, rc
            C.memmove(C.addressof(allw) + r * 160 * nwin, C.addressof(w), 160 * nwin)
        got, _ = eng.edwards_msm_combine(allw, ranks, n_shard)
        assert got == case.want
    return step


def precomp_step(holder, case, static_case):
    """static_case's points are the precomputation's; the dynamic terms are case's."""
    acc = [0] * len(case.pool.k)
    for i in range(static_case.n):
        acc[static_case.idx[i]] += static_case.ints[i]
    for i in range(case.n):
        acc[case.idx[i]] += case.ints[i]
    want = case.pool.times_base(sum(a * kk for a, kk in zip(acc, case.pool.k)))
    ss = [static_case.sb[32 * i:32 * i + 32] for i in range(static_case.n)]
    ds = [case.sb[32 * i:32 * i + 32] for i in range(case.n)]
    dp = [case.comp[32 * i:32 * i + 32] for i in range(case.n)]

    def step(eng):
        got = holder["pre"].vartime_mixed_multiscalar_mul(ss, ds, dp)
        assert got == want
    return step


# ---- 1. concurrent contexts -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pool(oracle):
    return Pool(oracle)


@pytest.fixture(scope="module")
def sigs(oracle):
    return SigCase(oracle, 3000, keys=257, seed=7, bad=1234)


def test_concurrent_contexts_different_sizes(oracle, pool, sigs):
    """Four contexts on device 0, one thread each, released together: vartime MSMs at 2^18 and 4096 (whose digit sorts
    need more shared memory than each other in one of the two sort kernels), 20000 extended points, c = 20 at n = 200
    through the bucket pipeline, verify_batch with its short scalars, msm_batch, and a precomputation with window tables,
    created inside its thread."""
    import curve25519_dalek_b200 as pkg
    big, mid, ext = MsmCase(pool, 1 << 18, 1), MsmCase(pool, 4096, 2), MsmCase(pool, 20000, 3)
    tiny, small = MsmCase(pool, 200, 4), MsmCase(pool, 1000, 5)
    statics = MsmCase(pool, 4096, 6)
    d_mid = on_device(mid.sb, mid.comp)
    d_big_ext = on_device(big.sb, big.ext)
    batch = MsmCase(pool, 40000, 8)
    holder = {}
    engines = [pkg.Engine(0) for _ in range(4)]

    def make_precomp(eng):
        if "pre" not in holder:
            eng.set_option("precomp_tables", 1)
            holder["pre"] = pkg.VartimeEdwardsPrecomputation([pool.enc[j].tobytes() for j in statics.idx], engine=eng)

    try:
        jobs = [
            ("A", engines[0], [("msm 2^18", msm_step(big)), ("msm 4096 dev", msm_step(mid, device=d_mid)),
                               ("msm 2^18 ext dev", msm_step(big, fmt=1, device=d_big_ext))]),
            ("B", engines[1], [("msm 4096", msm_step(mid)), ("msm 20000 ext", msm_step(ext, fmt=1)),
                               ("msm 200 c=20", msm_step(tiny, options=(("window_bits", 20), ("small_straus", 0)))),
                               ("msm 2^18 c=9", msm_step(big, options=(("window_bits", 9),)))]),
            ("C", engines[2], [("verify_batch", verify_batch_step(sigs)), ("verify_batch bad", verify_batch_step(sigs, bad=True)),
                               ("msm_batch", msm_batch_step(batch, [0, 5, 190, 1190, 1190, 40000])),
                               ("msm_batch ct", msm_batch_step(small, [0, 1, 100, 1000], constant_time=True))]),
            ("D", engines[3], [("precomp new", make_precomp), ("precomp msm", precomp_step(holder, small, statics)),
                               ("msm 20000", msm_step(ext)), ("msm 4096 c=16", msm_step(mid, options=(("window_bits", 16),)))]),
        ]
        run_threads(jobs, rounds=3)
    finally:
        if "pre" in holder:
            holder["pre"].close()
        for e in engines:
            e.close()


# ---- 2. every family's first use, concurrently ----------------------------------------------------------------------
def test_concurrent_first_use_of_every_family(oracle, pool, sigs):
    """One fresh context per entry-point family, all released at once, so the per-context tables and kernel attributes
    of signing, verify_each, X25519 keys, mul_batch, the double-base comb, hash to curve, Lizard, the codecs and scalar
    inversion are built while the other threads run."""
    import curve25519_dalek_b200 as pkg
    import h2c_oracle
    import lizard_oracle
    import x25519_oracle
    xo, ho, lo = x25519_oracle.load(), h2c_oracle.load(), lizard_oracle.load()
    rnd = random.Random(11)
    B = oracle.basepoint()

    # signing: 300 messages, one key each
    seeds = [rnd.randbytes(32) for _ in range(300)]
    msgs = [rnd.randbytes(rnd.randrange(0, 200)) for _ in range(300)]
    offs = np.zeros(301, dtype=np.uint64); offs[1:] = np.cumsum([len(m) for m in msgs])
    flat = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy()
    want_sigs = b"".join(oracle.sign(m, s) for m, s in zip(msgs, seeds))
    want_pks = b"".join(oracle.public_key(s) for s in seeds)

    def sign(eng):
        assert eng.sign_flat(b"".join(seeds), 300, flat, offs, 300) == want_sigs
        assert eng.verifying_keys(b"".join(seeds), 300) == want_pks

    # verify_each: the first 2048 of the shared signatures (257 keys: the plain path) and one altered message
    n_each = 2048
    want_each = [oracle.verify(m, sigs.sigs[64 * i:64 * i + 64], sigs.pks[32 * i:32 * i + 32])
                 for i, m in enumerate(sigs.bad_msgs[:n_each])]
    assert want_each.count(0) == n_each - 1

    def verify_each(eng):
        rc, res = eng.verify_each_flat(sigs.flat_bad, sigs.offs[:n_each + 1], sigs.sigs, sigs.pks, n_each)
        assert rc == 1 and res == want_each
        # 4 keys sign 128 each: the per-key comb tables
        rc, res = eng.verify_each_flat(comb_flat, comb_offs, comb_sigs, comb_pks, 512)
        assert rc == 0 and res == [0] * 512

    comb_seeds = [rnd.randbytes(32) for _ in range(4)]
    comb_msgs = [rnd.randbytes(32) for _ in range(512)]
    comb_sigs = b"".join(oracle.sign(m, comb_seeds[i % 4]) for i, m in enumerate(comb_msgs))
    comb_pks = b"".join(oracle.public_key(comb_seeds[i % 4]) for i in range(512))
    comb_offs = np.arange(0, 32 * 513, 32, dtype=np.uint64)
    comb_flat = np.frombuffer(b"".join(comb_msgs), dtype=np.uint8).copy()

    # X25519 public keys
    xk = [rnd.randbytes(32) for _ in range(500)]
    want_x = b"".join(xo.public_key(k) for k in xk)

    def x25519_keys(eng):
        assert eng.x25519_public_keys(b"".join(xk), 500) == want_x

    # mul_batch: s_i P_i over compressed pool points
    ms = [rnd.randrange(2**255).to_bytes(32, "little") for _ in range(300)]
    mj = [rnd.randrange(len(pool.k)) for _ in range(300)]
    want_mul = b"".join(pool.times_base(int.from_bytes(s, "little") * pool.k[j]) for s, j in zip(ms, mj))

    def mul_batch(eng):
        rc, got, _ = eng.mul_batch(b"".join(ms), 300, b"".join(pool.enc[j].tobytes() for j in mj), 300, 300)
        assert rc == 0 and got == want_mul

    # double-base comb: a_i G + b_i H for 4096 pairs
    G = oracle.ristretto_compress(oracle.scalarmul(rnd.randrange(L).to_bytes(32, "little"), B))
    H = oracle.ristretto_compress(oracle.scalarmul(rnd.randrange(L).to_bytes(32, "little"), B))
    da = b"".join(rnd.randrange(2**255).to_bytes(32, "little") for _ in range(4096))
    db = b"".join(rnd.randrange(2**255).to_bytes(32, "little") for _ in range(4096))
    rc, want_db = oracle.ristretto_double_base_batch(da, db, G, H)
    assert rc == 0

    def double_base(eng):
        rc, got = eng.ristretto_double_base_batch(da, db, G, H, 4096)
        assert rc == 0 and got == want_db

    # hash to curve (RFC 9380 ..._RO_)
    dst = b"QUUX-V01-CS02-with-edwards25519_XMD:SHA-512_ELL2_RO_"
    hmsgs = [rnd.randbytes(rnd.randrange(0, 100)) for _ in range(200)]
    want_h = b"".join(ho.flat_batch("hash_to_curve", hmsgs, dst))

    def hash_to_curve(eng):
        assert b"".join(pkg.EdwardsPoint.hash_to_curve_batch(hmsgs, dst, engine=eng)) == want_h

    # Lizard: encode, then decode back
    ldata = [rnd.randbytes(16) for _ in range(200)]
    want_l = lo.lizard_encode_batch(ldata)
    want_dec, want_status = lo.lizard_decode_batch(want_l)

    def lizard(eng):
        enc = eng.ristretto_lizard_encode_batch(b"".join(ldata), 200)
        assert enc == b"".join(want_l)
        rc, dec, status = eng.ristretto_lizard_decode_batch(enc, 200)
        assert rc == (0 if want_status == bytes(200) else 1) and status == want_status and dec == want_dec

    # codecs: decompress (with undecodable encodings among them) and compress back
    encs = [pool.enc[j].tobytes() for j in range(len(pool.k))] + [(2).to_bytes(32, "little"), rnd.randbytes(32)]
    dec = [oracle.decompress(e) for e in encs]
    want_ok = bytes(0 if p is None else 1 for p in dec)
    want_comp = b"".join(oracle.compress(oracle.identity() if p is None else p) for p in dec)

    def codecs(eng):
        rc, limbs, ok = eng.decompress_batch(b"".join(encs), len(encs))
        assert rc == 1 and ok == want_ok
        assert eng.compress_batch(limbs, len(encs)) == want_comp

    # scalar inversion
    inv_in = [rnd.randrange(1, L).to_bytes(32, "little") for _ in range(1000)]
    want_inv, want_prod = oracle.scalar_invert_batch(inv_in)

    def invert(eng):
        got, prod = eng.scalar_invert_batch(b"".join(inv_in), 1000)
        assert got == b"".join(want_inv) and prod == want_prod

    steps = [("sign", sign), ("verify_each", verify_each), ("x25519 keys", x25519_keys), ("mul_batch", mul_batch),
             ("double-base comb", double_base), ("hash_to_curve", hash_to_curve), ("lizard", lizard), ("codecs", codecs),
             ("invert", invert)]
    engines = [pkg.Engine(0) for _ in steps]
    try:
        run_threads([(label, e, [(label, fn)]) for e, (label, fn) in zip(engines, steps)], rounds=2)
    finally:
        for e in engines:
            e.close()


# ---- 3. one context, many entry points and sizes in turn -----------------------------------------------------------
def test_interleaved_calls_on_one_context(oracle, pool, sigs):
    """About 80 seeded calls on one context: MSM sizes going big -> small -> big over 0, 1, 189, 190, 4096, 2^16 + 3
    and 2^18 with window_bits, host_chunks, point format and host or device buffers changing between calls, and
    verify_batch, verify_batches, msm_batch and partial + combine in between.  A precomputation made early is used after
    later calls have regrown the workspaces it was made with."""
    import curve25519_dalek_b200 as pkg
    rnd = random.Random(2024)
    sizes = [0, 1, 189, 190, 4096, (1 << 16) + 3, 1 << 18]
    cases = {n: MsmCase(pool, n, 100 + n) for n in sizes}
    dev = {n: {fmt: on_device(cases[n].sb, cases[n].points(fmt)) for fmt in (0, 1)} for n in sizes if n}
    statics, dyn = MsmCase(pool, 5000, 31), MsmCase(pool, 150, 32)
    batch = MsmCase(pool, 36000, 33)
    order = sizes[::-1] + sizes[1:] + sizes[::-1][1:]          # big -> small -> big -> small
    schedule = []
    for n in order:
        for _ in range(3):
            fmt = rnd.randrange(2)
            opts = [("window_bits", rnd.choice([0, 0, 4, 7, 11, 13, 16, 20]) if n >= 190 or rnd.random() < 0.5 else 0),
                    ("host_chunks", rnd.randrange(1, 9))]
            device = dev[n][fmt] if n and rnd.random() < 0.4 else None
            if n and n < 190 and rnd.random() < 0.5:
                opts.append(("small_straus", 0))
            schedule.append(("msm n=%d fmt=%d %s %s" % (n, fmt, "dev" if device else "host", opts),
                             msm_step(cases[n], fmt=fmt, device=device, options=tuple(opts))))
        extra = rnd.choice(["verify_batch", "verify_batches", "msm_batch", "partial", "precomp"])
        if extra == "verify_batch":
            schedule.append((extra, verify_batch_step(sigs, bad=rnd.random() < 0.5)))
        elif extra == "verify_batches":
            schedule.append((extra, verify_batches_step(sigs, 256, sigs.want_batches[256])))
        elif extra == "msm_batch":
            schedule.append((extra, msm_batch_step(batch, [0, 3, 3, 190, 2000, 36000], fmt=rnd.randrange(2))))
        elif extra == "partial" and n >= 2:
            schedule.append(("partial+combine n=%d" % n, partial_combine_step(cases[n])))
    holder = {}
    eng = pkg.Engine(0)
    try:
        holder["pre"] = pkg.VartimeEdwardsPrecomputation([pool.enc[j].tobytes() for j in statics.idx], engine=eng)
        pre_step = precomp_step(holder, dyn, statics)
        pre_step(eng)
        # the precomputation is used again every so often, among the regrowing workspaces
        full = []
        for i, s in enumerate(schedule):
            full.append(s)
            if i % 10 == 9:
                full.append(("precomp", pre_step))
        full.append(("precomp", pre_step))
        assert 70 <= len(full) <= 100, len(full)
        failures = []
        for i, (label, fn) in enumerate(full):
            try:
                fn(eng)
            except Exception as exc:                        # noqa: BLE001
                failures.append("call %d (%s): %r; last_error=%r" % (i, label, exc, last_error(eng)))
        assert not failures, "\n".join(failures)
    finally:
        if "pre" in holder:
            holder["pre"].close()
        eng.close()


# ---- 4. two contexts in one thread ----------------------------------------------------------------------------------
def test_two_contexts_one_thread_sizes_and_options(pool):
    import curve25519_dalek_b200 as pkg
    big, small, hundred = MsmCase(pool, 1 << 18, 41), MsmCase(pool, 4096, 42), MsmCase(pool, 100, 43)
    a, b = pkg.Engine(0), pkg.Engine(0)
    try:
        for eng, case in ((a, big), (b, small), (a, small), (b, big)):
            rc, got, _ = eng.edwards_vartime_msm(case.sb, case.comp, case.n)
            assert rc == 0 and got == case.want, case.n

        def launches(eng):
            l0 = eng.launch_count()
            rc, got, _ = eng.edwards_vartime_msm(hundred.sb, hundred.comp, 100)
            assert rc == 0 and got == hundred.want
            return eng.launch_count() - l0

        b_before, a_before = launches(b), launches(a)
        assert b_before == a_before <= 5                     # the vartime Straus path
        a.set_option("small_straus", 0)
        b_after, a_after = launches(b), launches(a)
        assert b_after == b_before                           # B's options are its own
        b.set_option("small_straus", 0)
        try:
            assert a_after == launches(b) > 10              # A runs the bucket pipeline, as B does with the same option
        finally:
            b.set_option("small_straus", 1)
    finally:
        a.close()
        b.close()


# ---- 5. errors do not leak into later calls ---------------------------------------------------------------------------
def _right_after(a, b, case, sigs):
    for eng in (a, b):
        rc, got, _ = eng.edwards_vartime_msm(case.sb, case.comp, case.n)
        assert rc == 0 and got == case.want, last_error(eng)
        assert eng.verify_batch_flat(sigs.flat, sigs.offs, sigs.sigs, sigs.pks, sigs.n) == 0, last_error(eng)


def test_errors_on_one_context_leave_the_next_calls_right(pool, sigs):
    import curve25519_dalek_b200 as pkg
    case = MsmCase(pool, 3000, 51)
    a, b = pkg.Engine(0), pkg.Engine(0)
    try:
        # an argument error: RISTRETTO is not a point format of the Edwards MSM
        out = (C.c_uint8 * 32)()
        assert a.lib.dalek_b200_edwards_vartime_msm(a.h, case.sb, case.comp, 2, case.n, C.addressof(out), None) == -1
        _right_after(a, b, case, sigs)
        # an undecodable point: None
        bad = bytearray(case.comp); bad[32 * 17:32 * 18] = (2).to_bytes(32, "little")
        rc, _, _ = a.edwards_vartime_msm(case.sb, bytes(bad), case.n)
        assert rc == 1
        _right_after(a, b, case, sigs)
        # a failing batch verification
        assert a.verify_batch_flat(sigs.flat_bad, sigs.offs, sigs.sigs, sigs.pks, sigs.n) == 1
        _right_after(a, b, case, sigs)
    finally:
        a.close()
        b.close()


def test_failed_allocation_leaves_the_next_calls_right(pool, sigs):
    """2^40 wide scalars ask for 64 TiB of device memory: the first allocation fails, before any input byte is read, and
    the call returns DALEK_E_NOMEM.  The runtime's record of that failure must not reach the next call of the thread."""
    import curve25519_dalek_b200 as pkg
    case = MsmCase(pool, 3000, 52)
    a, b = pkg.Engine(0), pkg.Engine(0)
    try:
        tiny_in, tiny_out = (C.c_uint8 * 64)(), (C.c_uint8 * 32)()
        rc = a.lib.dalek_b200_scalar_from_wide_batch(a.h, C.addressof(tiny_in), 1 << 40, C.addressof(tiny_out))
        assert rc == -4, (rc, last_error(a))
        wide = random.Random(5).randbytes(64 * 10)
        want = b"".join(pyref.sc_bytes(int.from_bytes(wide[64 * i:64 * i + 64], "little") % L) for i in range(10))
        assert a.scalar_from_wide_batch(wide, 10) == want
        _right_after(a, b, case, sigs)
    finally:
        a.close()
        b.close()
