"""ctypes binding of libdalek_b200.so plus thin classes mirroring the reference's trait surface."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
POINTS_RISTRETTO = 2
POINTS_COMPRESSED = 0
POINTS_EXTENDED = 1
POINTS_MONTGOMERY = 3        # Montgomery u (an output format of Engine.mul_base_ct_batch)

_lib = None


def library_path():
    # DALEK_B200_LIB selects an alternative build of the same engine (tuning experiments only)
    return os.environ.get("DALEK_B200_LIB") or os.path.join(HERE, "libdalek_b200.so")


def load_library():
    """Load the CUDA engine.  Fails loudly if the extension has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError("libdalek_b200.so is missing: run `python -m curve25519_dalek_b200.build` "
                           "(or __graft_entry__.build()); there is no CPU fallback")
    lib = C.CDLL(path)
    vp, sz, u8p, u64p = C.c_void_p, C.c_size_t, C.c_char_p, C.c_void_p
    lib.dalek_b200_init.argtypes = [C.c_int, C.POINTER(vp)]
    lib.dalek_b200_destroy.argtypes = [vp]
    lib.dalek_b200_destroy.restype = None
    lib.dalek_b200_last_error.argtypes = [vp]
    lib.dalek_b200_last_error.restype = C.c_char_p
    lib.dalek_b200_set_option.argtypes = [vp, C.c_char_p, C.c_long]
    lib.dalek_b200_get_option.argtypes = [vp, C.c_char_p, C.POINTER(C.c_long)]
    lib.dalek_b200_launch_count.argtypes = [vp]
    lib.dalek_b200_launch_count.restype = C.c_uint64
    lib.dalek_b200_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.dalek_b200_last_call_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.dalek_b200_last_stage_ms.argtypes = [vp, C.c_char_p, C.POINTER(C.c_float)]
    for name in ("dalek_b200_edwards_vartime_msm", "dalek_b200_edwards_ct_msm", "dalek_b200_edwards_vartime_msm_dev"):
        getattr(lib, name).argtypes = [vp, vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_msm_window_count.argtypes = [vp, sz]
    lib.dalek_b200_edwards_msm_partial.argtypes = [vp, vp, vp, C.c_int, sz, sz, vp]
    lib.dalek_b200_edwards_msm_partial_dev.argtypes = [vp, vp, vp, C.c_int, sz, sz, vp]
    lib.dalek_b200_edwards_msm_combine.argtypes = [vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_edwards_msm_combine_dev.argtypes = [vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_edwards_msm_partial_async.argtypes = [vp, vp, vp, C.c_int, sz, sz, vp]
    lib.dalek_b200_edwards_msm_partial_dev_async.argtypes = [vp, vp, vp, C.c_int, sz, sz, vp]
    lib.dalek_b200_msm_partial_bytes.argtypes = [vp, sz]
    lib.dalek_b200_msm_partial_bytes.restype = sz
    lib.dalek_b200_stream.argtypes = [vp]
    lib.dalek_b200_stream.restype = vp
    lib.dalek_b200_init_multi.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    lib.dalek_b200_destroy_multi.argtypes = [vp]
    lib.dalek_b200_destroy_multi.restype = None
    lib.dalek_b200_multi_device_count.argtypes = [vp]
    lib.dalek_b200_multi_ctx.argtypes = [vp, C.c_int]
    lib.dalek_b200_multi_ctx.restype = vp
    lib.dalek_b200_multi_last_error.argtypes = [vp]
    lib.dalek_b200_multi_last_error.restype = C.c_char_p
    lib.dalek_b200_edwards_vartime_msm_multi.argtypes = [vp, vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_ristretto_double_base_batch.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.dalek_b200_ristretto_vartime_msm.argtypes = [vp, vp, vp, sz, vp]
    lib.ed25519_b200_verify_batch.argtypes = [vp, vp, vp, vp, vp, sz]
    lib.ed25519_b200_verify_batch_flat.argtypes = [vp, vp, vp, vp, vp, sz]
    lib.ed25519_b200_verify_batch_flat_dev.argtypes = [vp, vp, vp, vp, vp, sz, sz]
    lib.ed25519_b200_verify_batches_flat.argtypes = [vp, vp, vp, vp, vp, sz, sz, vp]
    lib.ed25519_b200_verify_batch_flat_points.argtypes = [vp, vp, vp, vp, vp, vp, sz]
    lib.ed25519_b200_verify_batch_flat_points_dev.argtypes = [vp, vp, vp, vp, vp, vp, sz]
    lib.ed25519_b200_verify_batches_flat_points.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, vp]
    lib.ed25519_b200_verify_batches_flat_points_dev.argtypes = [vp, vp, vp, vp, vp, vp, sz, sz, vp]
    lib.ed25519_b200_verify_batches_flat_dev.argtypes = [vp, vp, vp, vp, vp, sz, sz, vp]
    lib.dalek_b200_precomp_new.argtypes = [vp, vp, C.c_int, sz, C.POINTER(vp)]
    lib.dalek_b200_precomp_len.argtypes = [vp]
    lib.dalek_b200_precomp_len.restype = sz
    lib.dalek_b200_precomp_destroy.argtypes = [vp]
    lib.dalek_b200_precomp_destroy.restype = None
    lib.dalek_b200_precomp_mixed_msm.argtypes = [vp, vp, vp, sz, vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_basepoint_tables_new.argtypes = [vp, vp, C.c_int, sz, vp, C.POINTER(vp)]
    lib.dalek_b200_basepoint_tables_len.argtypes = [vp]
    lib.dalek_b200_basepoint_tables_len.restype = sz
    lib.dalek_b200_basepoint_tables_destroy.argtypes = [vp]
    lib.dalek_b200_basepoint_tables_destroy.restype = None
    lib.dalek_b200_basepoint_tables_basepoints.argtypes = [vp, vp, vp]
    lib.dalek_b200_basepoint_tables_mul.argtypes = [vp, vp, vp, vp, sz, C.c_int, vp]
    lib.dalek_b200_basepoint_tables_mul_dev.argtypes = [vp, vp, vp, vp, sz, C.c_int, vp]
    lib.dalek_b200_edwards_decompress_batch.argtypes = [vp, vp, sz, vp, vp]
    lib.dalek_b200_ristretto_decompress_batch.argtypes = [vp, vp, sz, vp, vp]
    lib.dalek_b200_edwards_compress_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_ristretto_double_and_compress_batch.argtypes = [vp, vp, sz, vp]
    lib.ed25519_b200_verify_each_flat.argtypes = [vp, vp, vp, vp, vp, sz, C.c_int, vp]
    lib.ed25519_b200_verify_each_flat_dev.argtypes = [vp, vp, vp, vp, vp, sz, C.c_int, vp]
    lib.dalek_b200_scalar_from_wide_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_scalar_invert_batch.argtypes = [vp, vp, sz, vp, vp]
    for name in ("dalek_b200_scalar_binary_batch", "dalek_b200_scalar_binary_batch_dev"):
        getattr(lib, name).argtypes = [vp, C.c_int, vp, sz, vp, sz, sz, vp]
    for name in ("dalek_b200_scalar_unary_batch", "dalek_b200_scalar_unary_batch_dev"):
        getattr(lib, name).argtypes = [vp, C.c_int, vp, sz, vp]
    lib.dalek_b200_scalar_from_bytes_batch.argtypes = [vp, vp, sz, C.c_int, vp, vp]
    lib.dalek_b200_scalar_hash_from_bytes_batch.argtypes = [vp, vp, vp, sz, vp]
    for name in ("dalek_b200_scalar_fold_batch", "dalek_b200_scalar_fold_batch_dev"):
        getattr(lib, name).argtypes = [vp, C.c_int, vp, vp, sz, vp]
    lib.ed25519_b200_last_zs.argtypes = [vp, vp, sz]
    lib.dalek_b200_edwards_mul_base_batch.argtypes = [vp, vp, sz, vp, vp]
    lib.ed25519_b200_sign_batch_flat.argtypes = [vp, vp, vp, vp, sz, vp, vp]
    lib.ed25519_b200_verifying_keys.argtypes = [vp, vp, sz, vp]
    lib.ed25519_b200_sign_flat.argtypes = [vp, vp, sz, vp, vp, sz, vp]
    lib.ed25519_b200_sign_prehashed.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp]
    lib.ed25519_b200_verify_prehashed_each.argtypes = [vp, vp, vp, sz, vp, vp, sz, C.c_int, vp]
    lib.ed25519_b200_key_set_new.argtypes = [vp, vp, sz, vp, vp, C.POINTER(vp)]
    lib.ed25519_b200_key_set_len.argtypes = [vp]
    lib.ed25519_b200_key_set_len.restype = sz
    lib.ed25519_b200_key_set_destroy.argtypes = [vp]
    lib.ed25519_b200_key_set_destroy.restype = None
    lib.ed25519_b200_key_set_verify_flat.argtypes = [vp, vp, vp, vp, vp, vp, sz, C.c_int, vp]
    lib.ed25519_b200_key_set_verify_flat_dev.argtypes = [vp, vp, vp, vp, vp, vp, sz, C.c_int, vp]
    lib.ed25519_b200_key_set_verify_prehashed.argtypes = [vp, vp, vp, vp, sz, vp, vp, sz, C.c_int, vp]
    lib.ed25519_b200_expanded_verifying_keys.argtypes = [vp, vp, sz, vp]
    lib.ed25519_b200_raw_sign_flat.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp]
    lib.ed25519_b200_raw_sign_prehashed.argtypes = [vp, vp, vp, sz, vp, sz, vp, sz, vp]
    lib.ed25519_b200_signing_key_set_new.argtypes = [vp, vp, sz, C.c_int, vp, C.POINTER(vp)]
    lib.ed25519_b200_signing_key_set_len.argtypes = [vp]
    lib.ed25519_b200_signing_key_set_len.restype = sz
    lib.ed25519_b200_signing_key_set_verifying_keys.argtypes = [vp, vp]
    lib.ed25519_b200_signing_key_set_destroy.argtypes = [vp]
    lib.ed25519_b200_signing_key_set_destroy.restype = None
    lib.ed25519_b200_signing_key_set_sign_flat.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.ed25519_b200_signing_key_set_sign_flat_dev.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.ed25519_b200_signing_key_set_sign_prehashed.argtypes = [vp, vp, vp, vp, sz, vp, sz, vp]
    lib.dalek_b200_edwards_to_montgomery_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_x25519_batch.argtypes = [vp, vp, vp, sz, vp, vp]
    lib.dalek_b200_x25519_batch_dev.argtypes = [vp, vp, vp, sz, vp, vp]
    lib.dalek_b200_x25519_public_keys.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_montgomery_mul_batch.argtypes = [vp, vp, sz, vp, sz, sz, vp]
    lib.dalek_b200_montgomery_mul_batch_dev.argtypes = [vp, vp, sz, vp, sz, sz, vp]
    lib.dalek_b200_montgomery_mul_bits_be_batch.argtypes = [vp, vp, sz, sz, sz, vp, sz, sz, vp]
    lib.dalek_b200_montgomery_to_edwards_batch.argtypes = [vp, vp, vp, sz, vp, vp]
    lib.dalek_b200_mul_base_ct_batch.argtypes = [vp, vp, sz, C.c_int, C.c_int, vp]
    lib.dalek_b200_mul_batch.argtypes = [vp, vp, sz, vp, C.c_int, sz, sz, C.c_int, vp, vp]
    lib.dalek_b200_mul_batch_dev.argtypes = [vp, vp, sz, vp, C.c_int, sz, sz, C.c_int, vp, vp]
    lib.dalek_b200_edwards_torsion_batch.argtypes = [vp, vp, C.c_int, sz, vp]
    lib.dalek_b200_vartime_double_base_batch.argtypes = [vp, vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_vartime_double_base_batch_dev.argtypes = [vp, vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_msm_batch.argtypes = [vp, vp, vp, C.c_int, vp, sz, C.c_int, vp, vp, vp]
    lib.dalek_b200_msm_batch_dev.argtypes = [vp, vp, vp, C.c_int, vp, sz, C.c_int, vp, vp, vp]
    lib.dalek_b200_ristretto_from_uniform_bytes_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_ristretto_hash_from_bytes_batch.argtypes = [vp, vp, vp, sz, vp]
    lib.dalek_b200_edwards_hash_to_curve_batch.argtypes = [vp, vp, vp, sz, vp, sz, vp]
    lib.dalek_b200_edwards_encode_to_curve_batch.argtypes = [vp, vp, vp, sz, vp, sz, vp]
    lib.dalek_b200_ristretto_map_to_curve_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_ristretto_lizard_encode_batch.argtypes = [vp, vp, sz, vp]
    lib.dalek_b200_ristretto_lizard_decode_batch.argtypes = [vp, vp, C.c_int, sz, vp, vp]
    lib.dalek_b200_ristretto_map_to_curve_inverse_batch.argtypes = [vp, vp, C.c_int, sz, vp, vp]
    for name in ("dalek_b200_point_add_batch", "dalek_b200_point_add_batch_dev"):
        getattr(lib, name).argtypes = [vp, vp, sz, vp, sz, C.c_int, sz, C.c_int, C.c_int, vp, vp]
    for name in ("dalek_b200_point_unary_batch", "dalek_b200_point_unary_batch_dev"):
        getattr(lib, name).argtypes = [vp, C.c_int, vp, C.c_int, sz, C.c_int, C.c_int, vp, vp]
    lib.dalek_b200_point_eq_batch.argtypes = [vp, vp, sz, vp, sz, C.c_int, sz, C.c_int, vp]
    for name in ("dalek_b200_point_sum_batch", "dalek_b200_point_sum_batch_dev"):
        getattr(lib, name).argtypes = [vp, vp, C.c_int, C.c_int, vp, sz, C.c_int, vp, vp]
    _lib = lib
    return lib


class EngineError(RuntimeError):
    pass


class SignatureError(Exception):
    """ed25519_dalek::SignatureError (ed25519-dalek/src/errors.rs:23-53): `.kind` is one of
    'Verify', 'ArrayLength', 'ScalarFormat', 'PointDecompression', 'PrehashedContextLength', 'MismatchedKeypair'."""
    KINDS = {1: "Verify", 2: "ArrayLength", 3: "ScalarFormat", 4: "PointDecompression", 5: "PrehashedContextLength",
             6: "MismatchedKeypair"}

    def __init__(self, code):
        self.code = code
        self.kind = self.KINDS.get(code, "Unknown")
        super().__init__(self.kind)


def _ptr(obj):
    """Host pointer of bytes / bytearray / numpy array / torch CPU tensor / int address."""
    if obj is None:
        return None
    if isinstance(obj, int):
        return obj
    if isinstance(obj, bytes):
        return C.cast(C.c_char_p(obj), C.c_void_p).value      # caller keeps `obj` alive across the call
    if isinstance(obj, bytearray):
        return C.addressof((C.c_char * len(obj)).from_buffer(obj)) if len(obj) else None
    if isinstance(obj, C.Array):
        return C.addressof(obj)
    if hasattr(obj, "data_ptr"):
        return obj.data_ptr()
    if hasattr(obj, "ctypes"):
        return obj.ctypes.data
    raise TypeError("unsupported buffer type %r" % type(obj))


class Engine:
    """One engine context bound to one CUDA device (dalek_b200_init)."""

    def __init__(self, device=0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.dalek_b200_init(device, C.byref(h))
        if rc != 0:
            raise EngineError("dalek_b200_init(device=%d) failed with %d: no usable sm_90 CUDA device "
                              "(the engine has no CPU fallback)" % (device, rc))
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.dalek_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise EngineError("engine error %d: %s" % (rc, self.lib.dalek_b200_last_error(self.h).decode()))
        return rc

    def set_option(self, name, value):
        self._check(self.lib.dalek_b200_set_option(self.h, name.encode(), int(value)))

    def get_option(self, name):
        v = C.c_long()
        self._check(self.lib.dalek_b200_get_option(self.h, name.encode(), C.byref(v)))
        return int(v.value)

    def launch_count(self):
        return int(self.lib.dalek_b200_launch_count(self.h))

    def last_call_ms(self):
        """Device time (CUDA events on the engine's stream) of the last MSM / verify_batch call, in ms."""
        ms = C.c_float()
        self.lib.dalek_b200_last_call_ms(self.h, C.byref(ms))
        return float(ms.value)

    def last_stage_ms(self, stage):
        """Device time of a named stage of the last call: 'bucket_accumulate' or 'decompress_R'."""
        ms = C.c_float()
        self._check(self.lib.dalek_b200_last_stage_ms(self.h, stage.encode(), C.byref(ms)))
        return float(ms.value)

    def last_kernel_ms(self):
        ms, n = C.c_float(), C.c_int()
        self.lib.dalek_b200_last_kernel_ms(self.h, C.byref(ms), C.byref(n))
        return ms.value, n.value

    # ---- MSM ----
    def edwards_vartime_msm(self, scalars, points, n, point_fmt=POINTS_COMPRESSED, device_ptrs=False, want_limbs=False):
        """Returns (rc, compressed32, limbs20 or None); rc 1 == None (a point did not decompress)."""
        out = (C.c_uint8 * 32)()
        limbs = (C.c_uint64 * 20)() if want_limbs else None
        fn = self.lib.dalek_b200_edwards_vartime_msm_dev if device_ptrs else self.lib.dalek_b200_edwards_vartime_msm
        keep = (scalars, points)
        rc = self._check(fn(self.h, _ptr(scalars), _ptr(points), point_fmt, n, C.addressof(out),
                            C.addressof(limbs) if want_limbs else None))
        del keep
        return rc, bytes(out), (list(limbs) if want_limbs else None)

    def edwards_ct_msm(self, scalars, points, n, point_fmt=POINTS_COMPRESSED, want_limbs=False):
        out = (C.c_uint8 * 32)()
        limbs = (C.c_uint64 * 20)() if want_limbs else None
        rc = self._check(self.lib.dalek_b200_edwards_ct_msm(self.h, _ptr(scalars), _ptr(points), point_fmt, n,
                                                            C.addressof(out), C.addressof(limbs) if want_limbs else None))
        return rc, bytes(out), (list(limbs) if want_limbs else None)

    # ---- sharded MSM: n_shard = size of the largest shard, the same on every rank (it selects the window width) ----
    def msm_window_count(self, n_shard):
        return self._check(self.lib.dalek_b200_msm_window_count(self.h, n_shard))

    def msm_partial_bytes(self, n_shard):
        """Bytes of a shard's device record (window accumulators + status word)."""
        return int(self.lib.dalek_b200_msm_partial_bytes(self.h, n_shard))

    def stream_ptr(self):
        """The context's main cudaStream_t as an integer (torch.cuda.ExternalStream(ptr))."""
        return int(self.lib.dalek_b200_stream(self.h) or 0)

    def edwards_msm_partial(self, scalars, points, n_local, n_shard, point_fmt=POINTS_COMPRESSED, device_ptrs=False):
        nwin = self.msm_window_count(n_shard)
        out = (C.c_uint64 * (20 * nwin))()
        fn = self.lib.dalek_b200_edwards_msm_partial_dev if device_ptrs else self.lib.dalek_b200_edwards_msm_partial
        rc = self._check(fn(self.h, _ptr(scalars), _ptr(points), point_fmt, n_local, n_shard, C.addressof(out)))
        return rc, out

    def edwards_msm_combine(self, windows, ranks, n_shard, want_limbs=False):
        out = (C.c_uint8 * 32)()
        limbs = (C.c_uint64 * 20)() if want_limbs else None
        self._check(self.lib.dalek_b200_edwards_msm_combine(self.h, _ptr(windows) if not isinstance(windows, C.Array) else C.addressof(windows),
                                                            ranks, n_shard, C.addressof(out),
                                                            C.addressof(limbs) if want_limbs else None))
        return bytes(out), (list(limbs) if want_limbs else None)

    def edwards_msm_partial_async(self, scalars, points, n_local, n_shard, d_out_record, point_fmt=POINTS_COMPRESSED,
                                  device_ptrs=False):
        """Enqueue the shard's MSM on the context's stream; its record lands in the device buffer d_out_record."""
        fn = self.lib.dalek_b200_edwards_msm_partial_dev_async if device_ptrs else self.lib.dalek_b200_edwards_msm_partial_async
        return self._check(fn(self.h, _ptr(scalars), _ptr(points), point_fmt, n_local, n_shard, _ptr(d_out_record)))

    def edwards_msm_combine_dev(self, d_records, ranks, n_shard, want_limbs=False):
        """(rc, compressed, limbs) from `ranks` gathered device records; rc 1 == None."""
        out = (C.c_uint8 * 32)()
        limbs = (C.c_uint64 * 20)() if want_limbs else None
        rc = self._check(self.lib.dalek_b200_edwards_msm_combine_dev(self.h, _ptr(d_records), ranks, n_shard, C.addressof(out),
                                                                     C.addressof(limbs) if want_limbs else None))
        return rc, bytes(out), (list(limbs) if want_limbs else None)

    # ---- Ristretto ----
    def ristretto_double_base_batch(self, a, b, G, H, n, out=None):
        """a_i*G + b_i*H for n pairs (host buffers).  With `out` (a writable 32*n-byte host buffer, e.g. a pinned
        tensor) the encodings are written there and `out` is returned instead of a bytes copy."""
        if out is not None:
            rc = self._check(self.lib.dalek_b200_ristretto_double_base_batch(self.h, _ptr(a), _ptr(b), _ptr(G), _ptr(H), n, _ptr(out)))
            return rc, out
        buf = (C.c_uint8 * (32 * max(n, 1)))()
        rc = self._check(self.lib.dalek_b200_ristretto_double_base_batch(self.h, _ptr(a), _ptr(b), _ptr(G), _ptr(H), n,
                                                                         C.addressof(buf)))
        return rc, bytes(buf)[:32 * n]

    def ristretto_vartime_msm(self, scalars, points, n):
        out = (C.c_uint8 * 32)()
        rc = self._check(self.lib.dalek_b200_ristretto_vartime_msm(self.h, _ptr(scalars), _ptr(points), n, C.addressof(out)))
        return rc, bytes(out)

    # ---- scalar batches ----
    def scalar_from_wide_batch(self, wide, n):
        """Scalar::from_bytes_mod_order_wide for n x 64 B -> n x 32 B."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_scalar_from_wide_batch(self.h, _ptr(wide), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def scalar_invert_batch(self, scalars, n):
        """Scalar::invert_batch: (inverses n x 32 B, product of all inverses)."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        prod = (C.c_uint8 * 32)()
        self._check(self.lib.dalek_b200_scalar_invert_batch(self.h, _ptr(scalars), n, C.addressof(out), C.addressof(prod)))
        return bytes(out)[:32 * n], bytes(prod)

    # ---- scalar arithmetic: canonical 32-byte scalars in and out; a non-canonical input raises EngineError ----
    SCALAR_BINARY_OPS = {"add": 0, "sub": 1, "mul": 2}
    SCALAR_UNARY_OPS = {"neg": 0, "invert": 1, "div_by_2": 2}
    SCALAR_FOLD_OPS = {"sum": 0, "product": 1}

    def _scalar_results(self, fn, args, n, device_ptrs, out):
        """Run a scalar call that writes n x 32 B: into `out` if given, else a new buffer (a CUDA tensor with device_ptrs,
        bytes otherwise)."""
        if device_ptrs:
            if out is None:
                import torch
                out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=torch.device("cuda", self.device))
            self._check(fn(self.h, *args, _ptr(out)))
            return out
        res = (C.c_uint8 * (32 * max(n, 1)))() if out is None else out
        self._check(fn(self.h, *args, _ptr(res)))
        return bytes(res)[:32 * n] if out is None else out

    def scalar_binary_batch(self, op, a, n_a, b, n_b, n, device_ptrs=False, out=None):
        """out[i] = A_i + B_i, A_i - B_i or A_i * B_i for op "add", "sub" or "mul" (dalek_b200_scalar_binary_batch): n_a and
        n_b are each 1 (broadcast) or n.  With device_ptrs every buffer is a device pointer or CUDA tensor, and `out` may be
        a non-broadcast input (in place)."""
        fn = self.lib.dalek_b200_scalar_binary_batch_dev if device_ptrs else self.lib.dalek_b200_scalar_binary_batch
        keep = (a, b)
        r = self._scalar_results(fn, (self.SCALAR_BINARY_OPS.get(op, op), _ptr(a), n_a, _ptr(b), n_b, n), n, device_ptrs, out)
        del keep
        return r

    def scalar_unary_batch(self, op, scalars, n, device_ptrs=False, out=None):
        """out[i] = -S_i, S_i^-1 (0 for 0) or S_i / 2 for op "neg", "invert" or "div_by_2" (dalek_b200_scalar_unary_batch);
        buffers as scalar_binary_batch."""
        fn = self.lib.dalek_b200_scalar_unary_batch_dev if device_ptrs else self.lib.dalek_b200_scalar_unary_batch
        return self._scalar_results(fn, (self.SCALAR_UNARY_OPS.get(op, op), _ptr(scalars), n), n, device_ptrs, out)

    def scalar_from_bytes_batch(self, data, n, canonical=False):
        """Scalar::from_bytes_mod_order, or from_canonical_bytes with `canonical`, for n x 32 B: (rc, n x 32 B, n ok bytes);
        rc 1 (DALEK_NONE) when a canonical decoding fails (its ok byte is 0 and its slot zero)."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        ok = (C.c_uint8 * max(n, 1))()
        rc = self._check(self.lib.dalek_b200_scalar_from_bytes_batch(self.h, _ptr(data), n, 1 if canonical else 0, C.addressof(out),
                                                                     C.addressof(ok)))
        return rc, bytes(out)[:32 * n], bytes(ok)[:n]

    def scalar_hash_from_bytes_batch(self, msgs_flat, offsets, n):
        """Scalar::hash_from_bytes::<Sha512> for n flat messages (layout of ristretto_hash_from_bytes_batch) -> n x 32 B."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_scalar_hash_from_bytes_batch(self.h, _ptr(msgs_flat), _ptr(offsets), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def scalar_fold_batch(self, op, scalars, offsets, m, device_ptrs=False, out=None):
        """Sum or Product (op "sum" or "product") of each segment offsets[j] .. offsets[j+1] of the flat scalars
        (dalek_b200_scalar_fold_batch): offsets are m + 1 uint64 starting at 0; an empty segment gives 0 or 1.  With
        device_ptrs scalars, offsets and the results are device buffers.  -> m x 32 B."""
        fn = self.lib.dalek_b200_scalar_fold_batch_dev if device_ptrs else self.lib.dalek_b200_scalar_fold_batch
        keep = (scalars, offsets)
        r = self._scalar_results(fn, (self.SCALAR_FOLD_OPS.get(op, op), _ptr(scalars), _ptr(offsets), m), m, device_ptrs, out)
        del keep
        return r

    # ---- batch codecs ----
    def decompress_batch(self, encodings, n, ristretto=False):
        """CompressedEdwardsY / CompressedRistretto decompress for n x 32 B: (rc, limbs [n x 20 u64], ok bytes)."""
        limbs = (C.c_uint64 * (20 * max(n, 1)))()
        ok = (C.c_uint8 * max(n, 1))()
        fn = self.lib.dalek_b200_ristretto_decompress_batch if ristretto else self.lib.dalek_b200_edwards_decompress_batch
        rc = self._check(fn(self.h, _ptr(encodings), n, C.addressof(limbs), C.addressof(ok)))
        return rc, limbs, bytes(ok)[:n]

    def compress_batch(self, limbs, n):
        """EdwardsPoint::compress_batch for n points given as 20 u64 limbs each -> n x 32 B."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_edwards_compress_batch(self.h, _ptr(limbs), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def ristretto_double_and_compress_batch(self, limbs, n):
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_ristretto_double_and_compress_batch(self.h, _ptr(limbs), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def edwards_to_montgomery_batch(self, limbs, n):
        """EdwardsPoint::to_montgomery_batch for n points given as 20 u64 limbs each -> n x 32 B (the identity gives 0)."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_edwards_to_montgomery_batch(self.h, _ptr(limbs), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    # ---- X25519 ----
    def x25519_batch(self, scalars, us, n, device_ptrs=False, want_contributory=False, out=None, contributory=None):
        """x25519(k_i, u_i) for n pairs of 32-byte secrets and u coordinates: (out, contributory or None).
        Host buffers give bytes.  With device_ptrs the inputs are device buffers (torch CUDA tensors or addresses); the
        results go to `out` / `contributory` if given (device buffers of 32 n and n bytes), else to new uint8 tensors on
        the engine's device, which are returned."""
        if device_ptrs:
            if out is None or (want_contributory and contributory is None):
                import torch
                dev = torch.device("cuda", self.device)
                if out is None:
                    out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=dev)
                if want_contributory and contributory is None:
                    contributory = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
            self._check(self.lib.dalek_b200_x25519_batch_dev(self.h, _ptr(scalars), _ptr(us), n, _ptr(out),
                                                             _ptr(contributory) if want_contributory else None))
            return out, (contributory if want_contributory else None)
        res = (C.c_uint8 * (32 * max(n, 1)))()
        flags = (C.c_uint8 * max(n, 1))() if want_contributory else None
        self._check(self.lib.dalek_b200_x25519_batch(self.h, _ptr(scalars), _ptr(us), n, C.addressof(res),
                                                     C.addressof(flags) if want_contributory else None))
        return bytes(res)[:32 * n], (bytes(flags)[:n] if want_contributory else None)

    def x25519_public_keys(self, scalars, n):
        """PublicKey::from(&StaticSecret) for n 32-byte secrets -> n x 32 B (constant-time fixed-base comb)."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_x25519_public_keys(self.h, _ptr(scalars), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    # ---- MontgomeryPoint ----
    def montgomery_mul_batch(self, scalars, n_scalars, us, n_points, n, device_ptrs=False, out=None):
        """Scalar * MontgomeryPoint (dalek_b200_montgomery_mul_batch): out[i] = u([s_i] P_i) for 32-byte scalars (bit 255
        clear, not clamped) and 32-byte u coordinates; n_scalars and n_points are each 1 (broadcast) or n.  Host buffers
        give bytes.  With device_ptrs the inputs are device buffers and the results go to `out` (32 n bytes), a new uint8
        tensor on the engine's device if not given, which is returned."""
        if device_ptrs:
            if out is None:
                import torch
                out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=torch.device("cuda", self.device))
            self._check(self.lib.dalek_b200_montgomery_mul_batch_dev(self.h, _ptr(scalars), n_scalars, _ptr(us), n_points, n,
                                                                     _ptr(out)))
            return out
        res = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_montgomery_mul_batch(self.h, _ptr(scalars), n_scalars, _ptr(us), n_points, n,
                                                             C.addressof(res)))
        return bytes(res)[:32 * n]

    def montgomery_mul_bits_be_batch(self, ints, int_bytes, n_ints, nbits, us, n_points, n):
        """MontgomeryPoint::mul_bits_be (dalek_b200_montgomery_mul_bits_be_batch): out[i] = u([b_i] P_i), b_i = bits
        nbits-1..0 of an int_bytes-byte little-endian integer (1 <= int_bytes <= 64, nbits <= 8 int_bytes); n_ints and
        n_points are each 1 (broadcast) or n.  Host buffers -> n x 32 B."""
        res = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_montgomery_mul_bits_be_batch(self.h, _ptr(ints), int_bytes, n_ints, nbits, _ptr(us),
                                                                     n_points, n, C.addressof(res)))
        return bytes(res)[:32 * n]

    def montgomery_to_edwards_batch(self, us, signs, n):
        """MontgomeryPoint::to_edwards (dalek_b200_montgomery_to_edwards_batch) for n u coordinates and n sign bytes:
        (rc, n x 32 B CompressedEdwardsY, n ok bytes); rc 1 (DALEK_NONE) when some item is None (ok 0, the identity's
        encoding in its slot)."""
        res = (C.c_uint8 * (32 * max(n, 1)))()
        ok = (C.c_uint8 * max(n, 1))()
        rc = self._check(self.lib.dalek_b200_montgomery_to_edwards_batch(self.h, _ptr(us), _ptr(signs), n, C.addressof(res),
                                                                         C.addressof(ok)))
        return rc, bytes(res)[:32 * n], bytes(ok)[:n]

    def mul_base_ct_batch(self, scalars, n, out_fmt=POINTS_COMPRESSED, clamped=False):
        """s_i B, constant time (dalek_b200_mul_base_ct_batch): out_fmt POINTS_COMPRESSED, POINTS_RISTRETTO or
        POINTS_MONTGOMERY; scalars with bit 255 clear, or any 32 bytes clamped (not with POINTS_RISTRETTO).  -> n x 32 B"""
        res = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_mul_base_ct_batch(self.h, _ptr(scalars), n, out_fmt, 1 if clamped else 0,
                                                          C.addressof(res)))
        return bytes(res)[:32 * n]

    # ---- variable-base scalar multiplication ----
    def mul_batch(self, scalars, n_scalars, points, n_points, n, point_fmt=POINTS_COMPRESSED, clamped=False, device_ptrs=False,
                  out=None, want_ok=False):
        """out[i] = s_i * P_i for n items (dalek_b200_mul_batch): n_scalars and n_points are each 1 (broadcast) or n.
        Returns (rc, out, ok or None); rc 1 (DALEK_NONE) when a point does not decode (its ok byte is 0 and its slot holds
        the identity).  Host buffers give bytes.  With device_ptrs the inputs are device buffers and the results go to
        `out` (32 n bytes) and, with want_ok, an n-byte ok buffer on the engine's device, new uint8 tensors if not given."""
        flags = 1 if clamped else 0
        if device_ptrs:
            ok = None
            if out is None or want_ok:
                import torch
                dev = torch.device("cuda", self.device)
                if out is None:
                    out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=dev)
                if want_ok:
                    ok = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
            rc = self._check(self.lib.dalek_b200_mul_batch_dev(self.h, _ptr(scalars), n_scalars, _ptr(points), point_fmt, n_points, n,
                                                               flags, _ptr(out), _ptr(ok)))
            return rc, out, ok
        res = (C.c_uint8 * (32 * max(n, 1)))() if out is None else out
        ok = (C.c_uint8 * max(n, 1))() if want_ok else None
        rc = self._check(self.lib.dalek_b200_mul_batch(self.h, _ptr(scalars), n_scalars, _ptr(points), point_fmt, n_points, n, flags,
                                                       _ptr(res), C.addressof(ok) if want_ok else None))
        return rc, (bytes(res)[:32 * n] if out is None else out), (bytes(ok)[:n] if want_ok else None)

    # ---- resident basepoint tables ----
    def basepoint_tables_new(self, points, k, point_fmt=POINTS_COMPRESSED):
        """dalek_b200_basepoint_tables_new: the comb tables of k points (k x 32-byte encodings, or k x 20 u64 limbs with
        POINTS_EXTENDED).  Returns (rc, handle or None, ok); rc 1 (DALEK_NONE) when a point does not decode (its ok byte
        is 0, and no handle is made)."""
        h = C.c_void_p()
        ok = (C.c_uint8 * max(k, 1))()
        rc = self._check(self.lib.dalek_b200_basepoint_tables_new(self.h, _ptr(points), point_fmt, k, C.addressof(ok), C.byref(h)))
        return rc, (h if h.value else None), bytes(ok)[:k]

    def basepoint_tables_len(self, handle):
        return int(self.lib.dalek_b200_basepoint_tables_len(handle))

    def basepoint_tables_destroy(self, handle):
        self.lib.dalek_b200_basepoint_tables_destroy(handle)

    def basepoint_tables_basepoints(self, handle):
        """The encodings of the k points of the handle, read back from their tables: k x 32 bytes."""
        k = self.basepoint_tables_len(handle)
        res = (C.c_uint8 * (32 * max(k, 1)))()
        self._check(self.lib.dalek_b200_basepoint_tables_basepoints(self.h, handle, C.addressof(res)))
        return bytes(res)[:32 * k]

    def basepoint_tables_mul(self, handle, scalars, indices, n, clamped=False, device_ptrs=False, out=None):
        """out[i] = s_i * P_{t_i} (dalek_b200_basepoint_tables_mul): indices holds n uint32 table indices, or None for
        table 0.  Host buffers give bytes.  With device_ptrs the inputs are device buffers and the results go to `out`
        (32 n bytes on the engine's device, a new uint8 tensor if not given)."""
        flags = 1 if clamped else 0
        if device_ptrs:
            if out is None:
                import torch
                out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=torch.device("cuda", self.device))
            self._check(self.lib.dalek_b200_basepoint_tables_mul_dev(self.h, handle, _ptr(scalars), _ptr(indices), n, flags,
                                                                     _ptr(out)))
            return out
        res = (C.c_uint8 * (32 * max(n, 1)))() if out is None else out
        self._check(self.lib.dalek_b200_basepoint_tables_mul(self.h, handle, _ptr(scalars), _ptr(indices), n, flags, _ptr(res)))
        return bytes(res)[:32 * n] if out is None else out

    # ---- variable-time double-base scalar multiplication ----
    def vartime_double_base_batch(self, ab, points, n, point_fmt=POINTS_COMPRESSED, device_ptrs=False, out=None, want_ok=False):
        """out[i] = a_i * A_i + b_i * B for n items (dalek_b200_vartime_double_base_batch): ab holds n pairs a_i || b_i of
        32-byte scalars (bit 255 clear), points the A_i.  Returns (rc, out, ok or None) like mul_batch; rc 1 (DALEK_NONE)
        when a point does not decode (its ok byte is 0 and its slot holds the identity).  With device_ptrs the inputs are
        device buffers and the results go to `out` (32 n bytes) and, with want_ok, an n-byte ok buffer on the engine's
        device, new uint8 tensors if not given."""
        if device_ptrs:
            ok = None
            if out is None or want_ok:
                import torch
                dev = torch.device("cuda", self.device)
                if out is None:
                    out = torch.empty(32 * max(n, 1), dtype=torch.uint8, device=dev)
                if want_ok:
                    ok = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
            rc = self._check(self.lib.dalek_b200_vartime_double_base_batch_dev(self.h, _ptr(ab), _ptr(points), point_fmt, n, _ptr(out),
                                                                               _ptr(ok)))
            return rc, out, ok
        res = (C.c_uint8 * (32 * max(n, 1)))() if out is None else out
        ok = (C.c_uint8 * max(n, 1))() if want_ok else None
        rc = self._check(self.lib.dalek_b200_vartime_double_base_batch(self.h, _ptr(ab), _ptr(points), point_fmt, n, _ptr(res),
                                                                       C.addressof(ok) if want_ok else None))
        return rc, (bytes(res)[:32 * n] if out is None else out), (bytes(ok)[:n] if want_ok else None)

    # ---- many independent MSMs ----
    def msm_batch(self, scalars, points, offsets, m, point_fmt=POINTS_COMPRESSED, constant_time=False, device_ptrs=False,
                  want_limbs=False):
        """m independent MSMs in one call (dalek_b200_msm_batch): MSM j is the sum of s_i * P_i over the terms
        offsets[j] .. offsets[j+1] of the flat scalars (32 B each) and points; offsets are m + 1 uint64.  With device_ptrs
        the three inputs are device buffers; the results always come back to the host.  Returns (rc, out, ok, limbs):
        m x 32 bytes of encodings (CompressedRistretto for Ristretto points, else CompressedEdwardsY), m ok bytes and,
        with want_limbs, m x 20 uint64.  rc 1 (DALEK_NONE): an MSM with ok 0 holds an undecodable point and its slot the
        identity.  constant_time raises EngineError for an undecodable point or a scalar with bit 255 set."""
        out = (C.c_uint8 * (32 * max(m, 1)))()
        ok = (C.c_uint8 * max(m, 1))()
        limbs = (C.c_uint64 * (20 * max(m, 1)))() if want_limbs else None
        fn = self.lib.dalek_b200_msm_batch_dev if device_ptrs else self.lib.dalek_b200_msm_batch
        keep = (scalars, points, offsets)
        rc = self._check(fn(self.h, _ptr(scalars), _ptr(points), point_fmt, _ptr(offsets), m, 1 if constant_time else 0,
                            C.addressof(out), C.addressof(limbs) if want_limbs else None, C.addressof(ok)))
        del keep
        return rc, bytes(out)[:32 * m], bytes(ok)[:m], (list(limbs)[:20 * m] if want_limbs else None)

    # ---- group operations ----
    def _point_results(self, fn, args, n, out_fmt, device_ptrs, out, want_ok):
        """Run a point call that writes n results in out_fmt (32 B, or 20 u64 for EXTENDED) and n ok bytes."""
        size = 160 if out_fmt == POINTS_EXTENDED else 32
        if device_ptrs:
            ok = None
            if out is None or want_ok:
                import torch
                dev = torch.device("cuda", self.device)
                if out is None:
                    out = torch.empty(size * max(n, 1), dtype=torch.uint8, device=dev)
                if want_ok:
                    ok = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
            rc = self._check(fn(self.h, *args, _ptr(out), _ptr(ok)))
            return rc, out, ok
        res = (C.c_uint8 * (size * max(n, 1)))() if out is None else out
        ok = (C.c_uint8 * max(n, 1))() if want_ok else None
        rc = self._check(fn(self.h, *args, _ptr(res), C.addressof(ok) if want_ok else None))
        return rc, (bytes(res)[:size * n] if out is None else out), (bytes(ok)[:n] if want_ok else None)

    @staticmethod
    def _point_flags(point_fmt, ristretto, sub=False):
        return (1 if sub else 0) | (2 if ristretto and point_fmt == POINTS_EXTENDED else 0)

    @staticmethod
    def _own_encoding(point_fmt, ristretto):
        return POINTS_RISTRETTO if point_fmt == POINTS_RISTRETTO or ristretto else POINTS_COMPRESSED

    def point_add_batch(self, a, n_a, b, n_b, n, point_fmt=POINTS_COMPRESSED, sub=False, ristretto=False, out_fmt=None,
                        device_ptrs=False, out=None, want_ok=False):
        """out[i] = A_i + B_i, or A_i - B_i with sub (dalek_b200_point_add_batch): n_a and n_b are each 1 (broadcast) or n.
        point_fmt COMPRESSED is Edwards, RISTRETTO Ristretto, EXTENDED Edwards unless `ristretto`.  out_fmt: the group's
        own encoding (the default) or POINTS_EXTENDED (n x 160 B of canonical limbs).  Returns (rc, out, ok or None) as
        mul_batch does; rc 1 (DALEK_NONE) when an input does not decode (its ok byte is 0 and its slot the identity)."""
        of = self._own_encoding(point_fmt, ristretto) if out_fmt is None else out_fmt
        fn = self.lib.dalek_b200_point_add_batch_dev if device_ptrs else self.lib.dalek_b200_point_add_batch
        keep = (a, b)
        r = self._point_results(fn, (_ptr(a), n_a, _ptr(b), n_b, point_fmt, n, self._point_flags(point_fmt, ristretto, sub), of),
                                n, of, device_ptrs, out, want_ok)
        del keep
        return r

    def point_unary_batch(self, op, points, n, point_fmt=POINTS_COMPRESSED, ristretto=False, out_fmt=None, device_ptrs=False,
                          out=None, want_ok=False):
        """out[i] = -P_i, 2 P_i or 8 P_i for op "neg", "double" or "mul_by_cofactor" (Edwards only)
        (dalek_b200_point_unary_batch); formats and results as point_add_batch."""
        ops = {"neg": 0, "double": 1, "mul_by_cofactor": 2}
        of = self._own_encoding(point_fmt, ristretto) if out_fmt is None else out_fmt
        fn = self.lib.dalek_b200_point_unary_batch_dev if device_ptrs else self.lib.dalek_b200_point_unary_batch
        return self._point_results(fn, (ops[op] if isinstance(op, str) else op, _ptr(points), point_fmt, n,
                                        self._point_flags(point_fmt, ristretto), of), n, of, device_ptrs, out, want_ok)

    def point_eq_batch(self, a, n_a, b, n_b, n, point_fmt=POINTS_COMPRESSED, ristretto=False):
        """eq | both_decoded << 1 per item (dalek_b200_point_eq_batch), the group's ct_eq; b = None compares with the identity.
        Returns (rc, n bytes); rc 1 when an input does not decode."""
        out = (C.c_uint8 * max(n, 1))()
        rc = self._check(self.lib.dalek_b200_point_eq_batch(self.h, _ptr(a), n_a, _ptr(b), n_b, point_fmt, n,
                                                            self._point_flags(point_fmt, ristretto), C.addressof(out)))
        return rc, bytes(out)[:n]

    def point_sum_batch(self, points, offsets, m, point_fmt=POINTS_COMPRESSED, ristretto=False, out_fmt=None, device_ptrs=False,
                        out=None, want_ok=False):
        """Sum of each segment offsets[j] .. offsets[j+1] of the flat points (dalek_b200_point_sum_batch): offsets are m + 1
        uint64 starting at 0.  Formats and results as point_add_batch (m results); an empty segment gives the identity, one
        with an undecodable point ok 0 and the identity.  With device_ptrs points, offsets and the results are device
        buffers."""
        of = self._own_encoding(point_fmt, ristretto) if out_fmt is None else out_fmt
        fn = self.lib.dalek_b200_point_sum_batch_dev if device_ptrs else self.lib.dalek_b200_point_sum_batch
        keep = (points, offsets)
        r = self._point_results(fn, (_ptr(points), point_fmt, self._point_flags(point_fmt, ristretto), _ptr(offsets), m, of), m, of,
                                device_ptrs, out, want_ok)
        del keep
        return r

    def torsion_batch(self, points, n, point_fmt=POINTS_COMPRESSED):
        """is_small_order | is_torsion_free << 1 | decoded << 2 per Edwards point (0 for an undecodable one), as bytes."""
        out = (C.c_uint8 * max(n, 1))()
        self._check(self.lib.dalek_b200_edwards_torsion_batch(self.h, _ptr(points), point_fmt, n, C.addressof(out)))
        return bytes(out)[:n]

    # ---- hash to group ----
    def ristretto_from_uniform_bytes_batch(self, data, n):
        """RistrettoPoint::from_uniform_bytes for n x 64 B -> n x 32 B CompressedRistretto."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_ristretto_from_uniform_bytes_batch(self.h, _ptr(data), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def ristretto_hash_from_bytes_batch(self, msgs_flat, offsets, n):
        """RistrettoPoint::hash_from_bytes::<Sha512> for n flat messages (message i = msgs_flat[offsets[i]:offsets[i+1]],
        n + 1 u64 offsets) -> n x 32 B CompressedRistretto."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_ristretto_hash_from_bytes_batch(self.h, _ptr(msgs_flat), _ptr(offsets), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def _edwards_h2c(self, fn, msgs_flat, offsets, n, dst):
        out = (C.c_uint8 * (32 * max(n, 1)))()
        dst = bytes(dst)
        self._check(fn(self.h, _ptr(msgs_flat), _ptr(offsets), n, _ptr(dst) if dst else None, len(dst), C.addressof(out)))
        return bytes(out)[:32 * n]

    def edwards_hash_to_curve_batch(self, msgs_flat, offsets, n, dst):
        """EdwardsPoint::hash_to_curve::<Sha512> (RFC 9380 ..._RO_) for n flat messages and one DST of 1..255 bytes
        -> n x 32 B CompressedEdwardsY."""
        return self._edwards_h2c(self.lib.dalek_b200_edwards_hash_to_curve_batch, msgs_flat, offsets, n, dst)

    def edwards_encode_to_curve_batch(self, msgs_flat, offsets, n, dst):
        """EdwardsPoint::encode_to_curve::<Sha512> (RFC 9380 ..._NU_), same layout as edwards_hash_to_curve_batch."""
        return self._edwards_h2c(self.lib.dalek_b200_edwards_encode_to_curve_batch, msgs_flat, offsets, n, dst)

    # ---- Lizard and the Elligator inverse ----
    def ristretto_map_to_curve_batch(self, data, n):
        """RistrettoPoint::map_to_curve for n x 32 B (bit 255 ignored) -> n x 32 B CompressedRistretto."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_ristretto_map_to_curve_batch(self.h, _ptr(data), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def ristretto_lizard_encode_batch(self, data, n):
        """RistrettoPoint::lizard_encode::<Sha256> for n x 16 B -> n x 32 B CompressedRistretto."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.dalek_b200_ristretto_lizard_encode_batch(self.h, _ptr(data), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def ristretto_lizard_decode_batch(self, points, n, point_fmt=POINTS_RISTRETTO):
        """RistrettoPoint::lizard_decode::<Sha256> for n points (RISTRETTO or EXTENDED).  Returns (rc, n x 16 B payloads,
        n status bytes: 0 Some, 1 None, 2 undecodable encoding); rc 1 (DALEK_NONE) unless every status is 0."""
        out = (C.c_uint8 * (16 * max(n, 1)))()
        st = (C.c_uint8 * max(n, 1))()
        rc = self._check(self.lib.dalek_b200_ristretto_lizard_decode_batch(self.h, _ptr(points), point_fmt, n, C.addressof(out),
                                                                           C.addressof(st)))
        return rc, bytes(out)[:16 * n], bytes(st)[:n]

    def ristretto_map_to_curve_inverse_batch(self, points, n, point_fmt=POINTS_RISTRETTO):
        """RistrettoPoint::map_to_curve_inverse for n points.  Returns (rc, n x 16 x 32 B candidates, list of n u16 masks);
        rc 1 (DALEK_NONE) when an encoding does not decode (its mask is 0)."""
        out = (C.c_uint8 * (512 * max(n, 1)))()
        mask = (C.c_uint16 * max(n, 1))()
        rc = self._check(self.lib.dalek_b200_ristretto_map_to_curve_inverse_batch(self.h, _ptr(points), point_fmt, n,
                                                                                  C.addressof(out), C.addressof(mask)))
        return rc, bytes(out)[:512 * n], list(mask)[:n]

    # ---- ed25519 ----
    def verify_batch_raw(self, messages, sigs, pubkeys):
        """messages: list of bytes; sigs: n*64 bytes; pubkeys: n*32 bytes.  Returns the C return code."""
        n = len(messages)
        bufs = [C.create_string_buffer(m, max(len(m), 1)) for m in messages]
        ptrs = (C.c_void_p * max(n, 1))(*[C.addressof(b) for b in bufs])
        lens = (C.c_size_t * max(n, 1))(*[len(m) for m in messages])
        return self._check(self.lib.ed25519_b200_verify_batch(self.h, C.addressof(ptrs), C.addressof(lens),
                                                              _ptr(sigs), _ptr(pubkeys), n))

    def verify_batch_flat(self, msgs_flat, offsets, sigs, pubkeys, n, device_ptrs=False, msgs_bytes=0):
        if device_ptrs:
            return self._check(self.lib.ed25519_b200_verify_batch_flat_dev(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs),
                                                                           _ptr(pubkeys), n, msgs_bytes))
        return self._check(self.lib.ed25519_b200_verify_batch_flat(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs),
                                                                   _ptr(pubkeys), n))

    def verify_batch_flat_points(self, msgs_flat, offsets, sigs, pubkeys, key_points, n, device_ptrs=False):
        """verify_batch for callers holding VerifyingKeys: key_points = n x 20 u64 limbs, the decompressed point of each key
        (E/verifying.rs:65-71); no key is decompressed inside the call."""
        fn = self.lib.ed25519_b200_verify_batch_flat_points_dev if device_ptrs else self.lib.ed25519_b200_verify_batch_flat_points
        return self._check(fn(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs), _ptr(pubkeys), _ptr(key_points), n))

    def verify_batches_flat(self, msgs_flat, offsets, sigs, pubkeys, n, batch_size, device_ptrs=False):
        """Independent batches of `batch_size` signatures in one call: (rc, verdicts) with verdicts[k] the result of
        verify_batch on batch k (0 Ok, 1 Verify, 3 ScalarFormat, 4 PointDecompression); rc = 0 iff all are 0."""
        nb = (n + batch_size - 1) // batch_size
        verdicts = (C.c_int32 * max(nb, 1))()
        fn = self.lib.ed25519_b200_verify_batches_flat_dev if device_ptrs else self.lib.ed25519_b200_verify_batches_flat
        rc = self._check(fn(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs), _ptr(pubkeys), n, batch_size, C.addressof(verdicts)))
        return rc, list(verdicts)[:nb]

    def verify_batches_flat_points(self, msgs_flat, offsets, sigs, pubkeys, key_points, n, batch_size, device_ptrs=False):
        """verify_batches_flat for callers holding VerifyingKeys (key_points = n x 20 u64 limbs): no key decompression."""
        nb = (n + batch_size - 1) // batch_size
        verdicts = (C.c_int32 * max(nb, 1))()
        fn = self.lib.ed25519_b200_verify_batches_flat_points_dev if device_ptrs else self.lib.ed25519_b200_verify_batches_flat_points
        rc = self._check(fn(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs), _ptr(pubkeys), _ptr(key_points), n, batch_size, C.addressof(verdicts)))
        return rc, list(verdicts)[:nb]

    def verify_each_flat(self, msgs_flat, offsets, sigs, pubkeys, n, strict=False, device_ptrs=False):
        """n independent verifications: (rc, results) with results[i] the code of VerifyingKey::verify (or verify_strict)
        for signature i alone; rc = 0 iff all are 0."""
        res = (C.c_uint8 * max(n, 1))()
        fn = self.lib.ed25519_b200_verify_each_flat_dev if device_ptrs else self.lib.ed25519_b200_verify_each_flat
        rc = self._check(fn(self.h, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs), _ptr(pubkeys), n, 1 if strict else 0, C.addressof(res)))
        return rc, list(res)[:n]

    def last_zs(self, n):
        out = (C.c_uint8 * (16 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_last_zs(self.h, C.addressof(out), n))
        return bytes(out)[:16 * n]

    # ---- synthesis ----
    def mul_base_batch(self, scalars, n, want_compressed=True):
        limbs = (C.c_uint64 * (20 * max(n, 1)))()
        comp = (C.c_uint8 * (32 * max(n, 1)))() if want_compressed else None
        self._check(self.lib.dalek_b200_edwards_mul_base_batch(self.h, _ptr(scalars), n, C.addressof(limbs),
                                                               C.addressof(comp) if want_compressed else None))
        return limbs, (bytes(comp)[:32 * n] if want_compressed else None)

    # ---- signing (secret keys; constant time) ----
    def verifying_keys(self, seeds, n):
        """SigningKey::from_bytes(seed).verifying_key() for n 32-byte seeds -> n x 32 B."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_verifying_keys(self.h, _ptr(seeds), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def sign_flat(self, seeds, n_seeds, msgs_flat, offsets, n):
        """Signer::try_sign for n flat messages with n_seeds = n keys (seed i signs message i) or 1 -> n x 64 B."""
        out = (C.c_uint8 * (64 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_sign_flat(self.h, _ptr(seeds), n_seeds, _ptr(msgs_flat), _ptr(offsets), n,
                                                    C.addressof(out)))
        return bytes(out)[:64 * n]

    def sign_prehashed(self, seeds, n_seeds, prehashes, n, context=None):
        """SigningKey::sign_prehashed (Ed25519ph) for n 64-byte prehashes and one context: (rc, n x 64 B); rc 5 is
        PrehashedContextLength (a context longer than 255 bytes)."""
        out = (C.c_uint8 * (64 * max(n, 1)))()
        ctx = bytes(context) if context is not None else b""
        rc = self._check(self.lib.ed25519_b200_sign_prehashed(self.h, _ptr(seeds), n_seeds, _ptr(prehashes), n,
                                                              _ptr(ctx) if ctx else None, len(ctx), C.addressof(out)))
        return rc, bytes(out)[:64 * n]

    def verify_prehashed_each(self, prehashes, sigs, pubkeys, n, context=None, strict=False):
        """verify_prehashed (or verify_prehashed_strict) of n signatures over 64-byte prehashes with one context:
        (rc, results) as in verify_each_flat."""
        res = (C.c_uint8 * max(n, 1))()
        ctx = bytes(context) if context is not None else b""
        rc = self._check(self.lib.ed25519_b200_verify_prehashed_each(self.h, _ptr(prehashes), _ptr(ctx) if ctx else None, len(ctx),
                                                                     _ptr(sigs), _ptr(pubkeys), n, 1 if strict else 0,
                                                                     C.addressof(res)))
        return rc, list(res)[:n]

    # ---- resident verifying-key sets ----
    def key_set_new(self, pubkeys, k):
        """ed25519_b200_key_set_new for k 32-byte keys: (rc, handle or None, ok, weak); rc 4 (PointDecompression) when a
        key does not decode (its ok byte is 0, and no handle is made)."""
        h = C.c_void_p()
        ok, weak = (C.c_uint8 * max(k, 1))(), (C.c_uint8 * max(k, 1))()
        rc = self._check(self.lib.ed25519_b200_key_set_new(self.h, _ptr(pubkeys), k, C.addressof(ok), C.addressof(weak), C.byref(h)))
        return rc, (h if h.value else None), bytes(ok)[:k], bytes(weak)[:k]

    def key_set_len(self, handle):
        return int(self.lib.ed25519_b200_key_set_len(handle))

    def key_set_destroy(self, handle):
        self.lib.ed25519_b200_key_set_destroy(handle)

    def key_set_verify_flat(self, handle, msgs_flat, offsets, sigs, indices, n, strict=False, device_ptrs=False):
        """verify (or verify_strict) of signature i under key indices[i] of the set (n uint32, or None for key 0):
        (rc, results) as in verify_each_flat.  With device_ptrs every input is a device buffer."""
        res = (C.c_uint8 * max(n, 1))()
        fn = self.lib.ed25519_b200_key_set_verify_flat_dev if device_ptrs else self.lib.ed25519_b200_key_set_verify_flat
        rc = self._check(fn(self.h, handle, _ptr(msgs_flat), _ptr(offsets), _ptr(sigs), _ptr(indices), n, 1 if strict else 0,
                            C.addressof(res)))
        return rc, list(res)[:n]

    def key_set_verify_prehashed(self, handle, prehashes, sigs, indices, n, context=None, strict=False):
        """verify_prehashed (or verify_prehashed_strict) of signature i under key indices[i] of the set: (rc, results) as
        in verify_prehashed_each."""
        res = (C.c_uint8 * max(n, 1))()
        ctx = bytes(context) if context is not None else b""
        rc = self._check(self.lib.ed25519_b200_key_set_verify_prehashed(self.h, handle, _ptr(prehashes), _ptr(ctx) if ctx else None,
                                                                        len(ctx), _ptr(sigs), _ptr(indices), n,
                                                                        1 if strict else 0, C.addressof(res)))
        return rc, list(res)[:n]

    # ---- hazmat signing from ExpandedSecretKey bytes ----
    def expanded_verifying_keys(self, esks, n):
        """VerifyingKey::from(&ExpandedSecretKey::from_bytes(esk)) for n 64-byte esks -> n x 32 B."""
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_expanded_verifying_keys(self.h, _ptr(esks), n, C.addressof(out)))
        return bytes(out)[:32 * n]

    def raw_sign_flat(self, esks, vks, n_keys, msgs_flat, offsets, n):
        """hazmat::raw_sign for n flat messages with n_keys = n or 1 (esk, verifying key) pairs -> n x 64 B."""
        out = (C.c_uint8 * (64 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_raw_sign_flat(self.h, _ptr(esks), _ptr(vks), n_keys, _ptr(msgs_flat), _ptr(offsets), n,
                                                        C.addressof(out)))
        return bytes(out)[:64 * n]

    def raw_sign_prehashed(self, esks, vks, n_keys, prehashes, n, context=None):
        """hazmat::raw_sign_prehashed (Ed25519ph) for n 64-byte prehashes and one context: (rc, n x 64 B); rc 5 is
        PrehashedContextLength."""
        out = (C.c_uint8 * (64 * max(n, 1)))()
        ctx = bytes(context) if context is not None else b""
        rc = self._check(self.lib.ed25519_b200_raw_sign_prehashed(self.h, _ptr(esks), _ptr(vks), n_keys, _ptr(prehashes), n,
                                                                  _ptr(ctx) if ctx else None, len(ctx), C.addressof(out)))
        return rc, bytes(out)[:64 * n]

    # ---- resident signing-key sets ----
    def signing_key_set_new(self, keys, k, form):
        """ed25519_b200_signing_key_set_new for k keys of form SIGNING_KEY_SEED / _KEYPAIR / _EXPANDED: (rc, handle or None,
        status); rc 4 (PointDecompression) or 6 (MismatchedKeypair) is the status of the first failing keypair, and no
        handle is made."""
        h = C.c_void_p()
        status = (C.c_uint8 * max(k, 1))()
        rc = self._check(self.lib.ed25519_b200_signing_key_set_new(self.h, _ptr(keys), k, form, C.addressof(status), C.byref(h)))
        return rc, (h if h.value else None), bytes(status)[:k]

    def signing_key_set_len(self, handle):
        return int(self.lib.ed25519_b200_signing_key_set_len(handle))

    def signing_key_set_verifying_keys(self, handle):
        k = self.signing_key_set_len(handle)
        out = (C.c_uint8 * (32 * max(k, 1)))()
        self._check(self.lib.ed25519_b200_signing_key_set_verifying_keys(handle, C.addressof(out)))
        return bytes(out)[:32 * k]

    def signing_key_set_destroy(self, handle):
        self.lib.ed25519_b200_signing_key_set_destroy(handle)

    def signing_key_set_sign_flat(self, handle, msgs_flat, offsets, indices, n, device_ptrs=False, out=None):
        """Signer::try_sign of message i under key indices[i] of the set (n uint32, or None for key 0) -> n x 64 B.  With
        device_ptrs every buffer, `out` included, is a device pointer and the call returns None."""
        if device_ptrs:
            self._check(self.lib.ed25519_b200_signing_key_set_sign_flat_dev(self.h, handle, _ptr(msgs_flat), _ptr(offsets),
                                                                            _ptr(indices), n, _ptr(out)))
            return None
        res = (C.c_uint8 * (64 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_signing_key_set_sign_flat(self.h, handle, _ptr(msgs_flat), _ptr(offsets), _ptr(indices),
                                                                    n, C.addressof(res)))
        return bytes(res)[:64 * n]

    def signing_key_set_sign_prehashed(self, handle, prehashes, indices, n, context=None):
        """SigningKey::sign_prehashed of prehash i under key indices[i] of the set: (rc, n x 64 B); rc 5 is
        PrehashedContextLength."""
        res = (C.c_uint8 * (64 * max(n, 1)))()
        ctx = bytes(context) if context is not None else b""
        rc = self._check(self.lib.ed25519_b200_signing_key_set_sign_prehashed(self.h, handle, _ptr(prehashes),
                                                                              _ptr(ctx) if ctx else None, len(ctx), _ptr(indices),
                                                                              n, C.addressof(res)))
        return rc, bytes(res)[:64 * n]

    def sign_batch_flat(self, seeds, msgs_flat, offsets, n):
        pks = (C.c_uint8 * (32 * max(n, 1)))()
        sigs = (C.c_uint8 * (64 * max(n, 1)))()
        self._check(self.lib.ed25519_b200_sign_batch_flat(self.h, _ptr(seeds), _ptr(msgs_flat), _ptr(offsets), n,
                                                          C.addressof(pks), C.addressof(sigs)))
        return bytes(pks)[:32 * n], bytes(sigs)[:64 * n]


class MultiEngine:
    """One MSM over several GPUs of this node from a single process (dalek_b200_init_multi): contiguous shards, peer
    copies of the window-accumulator records to the first device, combine there."""

    def __init__(self, devices):
        self.lib = load_library()
        devs = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        rc = self.lib.dalek_b200_init_multi(devs, len(devices), C.byref(h))
        if rc != 0:
            raise EngineError("dalek_b200_init_multi(%r) failed with %d (the engine has no CPU fallback)" % (list(devices), rc))
        self.h = h
        self.devices = list(devices)

    def close(self):
        if getattr(self, "h", None):
            self.lib.dalek_b200_destroy_multi(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, name, value):
        for i in range(len(self.devices)):
            rc = self.lib.dalek_b200_set_option(self.lib.dalek_b200_multi_ctx(self.h, i), name.encode(), int(value))
            if rc:
                raise EngineError("set_option(%s) failed" % name)

    def last_call_ms(self):
        ms = C.c_float()
        self.lib.dalek_b200_last_call_ms(self.lib.dalek_b200_multi_ctx(self.h, 0), C.byref(ms))
        return float(ms.value)

    def edwards_vartime_msm(self, scalars, points, n, point_fmt=POINTS_COMPRESSED, want_limbs=False):
        """(rc, compressed32, limbs20 or None) like Engine.edwards_vartime_msm, host buffers."""
        out = (C.c_uint8 * 32)()
        limbs = (C.c_uint64 * 20)() if want_limbs else None
        keep = (scalars, points)
        rc = self.lib.dalek_b200_edwards_vartime_msm_multi(self.h, _ptr(scalars), _ptr(points), point_fmt, n, C.addressof(out),
                                                           C.addressof(limbs) if want_limbs else None)
        del keep
        if rc < 0:
            raise EngineError("engine error %d: %s" % (rc, self.lib.dalek_b200_multi_last_error(self.h).decode()))
        return rc, bytes(out), (list(limbs) if want_limbs else None)


_default = None


def default_engine():
    global _default
    if _default is None:
        _default = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    return _default


def _msm_batch(scalar_lists, point_lists, fmt, constant_time, engine):
    import array
    scalar_lists, point_lists = [list(s) for s in scalar_lists], [list(p) for p in point_lists]
    assert len(scalar_lists) == len(point_lists), "one point list per scalar list"
    for s, p in zip(scalar_lists, point_lists):
        # both iterators must have equal, exact sizes (edwards.rs:982-988, :1013-1019 assert)
        assert len(s) == len(p), "scalars and points must have the same length"
    m = len(scalar_lists)
    # a None among the points makes that MSM None; it is sent as an empty one
    none = [any(q is None for q in p) for p in point_lists]
    if constant_time and any(none):
        raise ValueError("multiscalar_mul takes points, not Options")
    offs = array.array("Q", [0])
    for s, skip in zip(scalar_lists, none):
        offs.append(offs[-1] + (0 if skip else len(s)))
    flat_s = b"".join(b"".join(s) for s, skip in zip(scalar_lists, none) if not skip)
    flat_p = b"".join(b"".join(p) for p, skip in zip(point_lists, none) if not skip)
    eng = engine or default_engine()
    rc, out, ok, _ = eng.msm_batch(flat_s, flat_p, offs.tobytes(), m, point_fmt=fmt, constant_time=constant_time)
    return [None if (skip or not ok[j]) else out[32 * j:32 * j + 32] for j, skip in enumerate(none)]


def _expect_all(results):
    if any(r is None for r in results):
        raise ValueError("should return some point")
    return results


def _point_binary(a, b, fmt, sub, engine):
    single_a, as_ = _items(a, 32, "points")
    single_b, bs = _items(b, 32, "points")
    n = _broadcast_len(single_a, as_, single_b, bs)
    if n == 0:
        return []
    eng = engine or default_engine()
    rc, raw, _ = eng.point_add_batch(b"".join(as_), len(as_), b"".join(bs), len(bs), n, fmt, sub=sub)
    if rc == 1:
        raise ValueError("a point does not decode")
    outs = [raw[32 * i:32 * i + 32] for i in range(n)]
    return outs[0] if single_a and single_b else outs


def _point_unary(points, op, fmt, engine):
    single, ps = _items(points, 32, "points")
    if not ps:
        return []
    eng = engine or default_engine()
    rc, raw, _ = eng.point_unary_batch(op, b"".join(ps), len(ps), fmt)
    if rc == 1:
        raise ValueError("a point does not decode")
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ps))]
    return outs[0] if single else outs


def _point_eq(a, b, fmt, engine):
    single_a, as_ = _items(a, 32, "points")
    if b is None:
        single_b, bs = True, []
        n = len(as_)
    else:
        single_b, bs = _items(b, 32, "points")
        n = _broadcast_len(single_a, as_, single_b, bs)
    if n == 0:
        return []
    eng = engine or default_engine()
    rc, flags = eng.point_eq_batch(b"".join(as_), len(as_), b"".join(bs) if b is not None else None, len(bs), n, fmt)
    if rc == 1:
        raise ValueError("a point does not decode")
    outs = [bool(f & 1) for f in flags]
    return outs[0] if single_a and single_b else outs


def _point_sum_batch(point_lists, fmt, engine):
    import array
    lists = [_items(list(p), 32, "points")[1] for p in point_lists]
    m = len(lists)
    if m == 0:
        return []
    offs = array.array("Q", [0])
    for p in lists:
        offs.append(offs[-1] + len(p))
    eng = engine or default_engine()
    rc, raw, _ = eng.point_sum_batch(b"".join(b"".join(p) for p in lists), offs.tobytes(), m, fmt)
    if rc == 1:
        raise ValueError("a point does not decode")
    return [raw[32 * j:32 * j + 32] for j in range(m)]


class _GroupOps:
    """The group operators (edwards.rs:786-876, ristretto.rs:809-908) on 32-byte encodings of the class's group, one thread
    per item on the GPU.  One item (bytes) gives one result, a list gives the list; in the binary forms a single item is
    used for every item of the other operand.  An undecodable encoding raises ValueError."""
    _FMT = None

    @classmethod
    def add_batch(cls, a, b, engine=None):
        """Add: A + B."""
        return _point_binary(a, b, cls._FMT, False, engine)

    @classmethod
    def sub_batch(cls, a, b, engine=None):
        """Sub: A - B."""
        return _point_binary(a, b, cls._FMT, True, engine)

    @classmethod
    def neg_batch(cls, points, engine=None):
        """Neg: -P."""
        return _point_unary(points, "neg", cls._FMT, engine)

    @classmethod
    def double_batch(cls, points, engine=None):
        """Group::double: 2P."""
        return _point_unary(points, "double", cls._FMT, engine)

    @classmethod
    def eq_batch(cls, a, b, engine=None):
        """ConstantTimeEq / PartialEq of the group (not of the bytes): a bool per item."""
        return _point_eq(a, b, cls._FMT, engine)

    @classmethod
    def is_identity_batch(cls, points, engine=None):
        """IsIdentity (traits.rs:33-48): a bool per item."""
        return _point_eq(points, None, cls._FMT, engine)

    @classmethod
    def sum(cls, points, engine=None):
        """Sum<T> (edwards.rs:837-851, ristretto.rs:882-892): the fold of the points from the identity."""
        return _point_sum_batch([list(points)], cls._FMT, engine)[0]

    @classmethod
    def sum_batch(cls, point_lists, engine=None):
        """Sum of each list of points, one call for all lists: the list of results (the identity for an empty list)."""
        return _point_sum_batch(point_lists, cls._FMT, engine)


class EdwardsPoint(_GroupOps):
    """Mirror of the trait impls on curve25519_dalek::edwards::EdwardsPoint.  Points are handled in
    their 32-byte CompressedEdwardsY encoding; results are returned compressed."""
    _FMT = POINTS_COMPRESSED

    @staticmethod
    def mul_by_cofactor_batch(points, engine=None):
        """EdwardsPoint::mul_by_cofactor (edwards.rs:1365-1367): 8P."""
        return _point_unary(points, "mul_by_cofactor", POINTS_COMPRESSED, engine)

    @staticmethod
    def optional_multiscalar_mul(scalars, points, engine=None):
        """VartimeMultiscalarMul::optional_multiscalar_mul (traits.rs:196-200): `points` holds 32-byte
        encodings; an entry that is None or fails to decompress makes the result None."""
        scalars, points = list(scalars), list(points)
        # both iterators must have equal, exact sizes (edwards.rs:1013-1019 asserts)
        assert len(scalars) == len(points), "scalars and points must have the same length"
        if any(p is None for p in points):
            return None
        eng = engine or default_engine()
        rc, comp, _ = eng.edwards_vartime_msm(b"".join(scalars), b"".join(points), len(scalars))
        return None if rc == 1 else comp

    @staticmethod
    def vartime_multiscalar_mul(scalars, points, engine=None):
        """traits.rs:249-262: .expect() on the optional form."""
        r = EdwardsPoint.optional_multiscalar_mul(scalars, points, engine)
        if r is None:
            raise ValueError("should return some point")
        return r

    @staticmethod
    def multiscalar_mul(scalars, points, engine=None):
        """MultiscalarMul::multiscalar_mul (traits.rs:128-133, edwards.rs:970-995), constant-time contract."""
        scalars, points = list(scalars), list(points)
        assert len(scalars) == len(points), "scalars and points must have the same length"
        eng = engine or default_engine()
        rc, comp, _ = eng.edwards_ct_msm(b"".join(scalars), b"".join(points), len(scalars))
        return comp

    @staticmethod
    def optional_multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        """optional_multiscalar_mul (traits.rs:196-262) for many independent MSMs in one call: item j is the MSM of
        scalar_lists[j] over point_lists[j] (CompressedEdwardsY).  Returns the list of 32-byte encodings, None where a
        point is None or does not decompress."""
        return _msm_batch(scalar_lists, point_lists, POINTS_COMPRESSED, False, engine)

    @staticmethod
    def vartime_multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        """traits.rs:249-262 for every item of optional_multiscalar_mul_batch: .expect() on each."""
        return _expect_all(_msm_batch(scalar_lists, point_lists, POINTS_COMPRESSED, False, engine))

    @staticmethod
    def multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        """MultiscalarMul::multiscalar_mul (traits.rs:78-134, edwards.rs:970-995) for many independent MSMs in one call,
        constant time in the scalars.  An undecodable point or a scalar with bit 255 set raises EngineError."""
        return _msm_batch(scalar_lists, point_lists, POINTS_COMPRESSED, True, engine)

    @staticmethod
    def to_montgomery_batch(limbs, n=None, engine=None):
        """EdwardsPoint::to_montgomery_batch (edwards.rs:592-612): `limbs` holds n points as 20 u64 radix-2^51 limbs
        each (X | Y | Z | T, e.g. what Engine.mul_base_batch returns); returns the n 32-byte Montgomery u coordinates."""
        n = len(limbs) // 20 if n is None else n
        eng = engine or default_engine()
        raw = eng.edwards_to_montgomery_batch(limbs, n)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    @staticmethod
    def mul_batch(scalars, points, engine=None):
        """EdwardsPoint * Scalar (edwards.rs:890-899) for each pair of a 32-byte scalar (bit 255 clear) and a 32-byte
        CompressedEdwardsY; a single scalar or a single point is used for every item.  Returns the CompressedEdwardsY of
        the product, or the list.  An undecodable point raises ValueError."""
        return _mul_batch(scalars, points, POINTS_COMPRESSED, False, engine)

    @staticmethod
    def mul_clamped_batch(bytes_list, points, engine=None):
        """EdwardsPoint::mul_clamped (edwards.rs:932-941): any 32 bytes, clamped and not reduced; broadcast as mul_batch."""
        return _mul_batch(bytes_list, points, POINTS_COMPRESSED, True, engine)

    @staticmethod
    def mul_base_batch(scalars, engine=None):
        """EdwardsPoint::mul_base (edwards.rs:918-928) for each 32-byte scalar (bit 255 clear, not reduced: the point is
        (s mod l) B), constant time at every batch size.  Returns the CompressedEdwardsY, or the list."""
        return _mul_base_batch(scalars, POINTS_COMPRESSED, False, engine)

    @staticmethod
    def mul_base_clamped_batch(bytes_list, engine=None):
        """EdwardsPoint::mul_base_clamped (edwards.rs:944-957): any 32 bytes, clamped and not reduced; like mul_base_batch."""
        return _mul_base_batch(bytes_list, POINTS_COMPRESSED, True, engine)

    @staticmethod
    def vartime_double_scalar_mul_basepoint_batch(a_list, points, b_list, engine=None):
        """EdwardsPoint::vartime_double_scalar_mul_basepoint (edwards.rs:1078-1087) for each item: a_i * A_i + b_i * B with
        32-byte scalars (bit 255 clear, not reduced) and CompressedEdwardsY points A_i.  Returns the list of 32-byte
        CompressedEdwardsY results.  An undecodable point raises ValueError.  Variable time."""
        return _double_base_batch(a_list, points, b_list, POINTS_COMPRESSED, engine)

    @staticmethod
    def is_small_order_batch(points, engine=None):
        """EdwardsPoint::is_small_order (edwards.rs:1405-1407) of each CompressedEdwardsY: a list of bool."""
        return [bool(f & 1) for f in _torsion_flags(points, engine)]

    @staticmethod
    def is_torsion_free_batch(points, engine=None):
        """EdwardsPoint::is_torsion_free (edwards.rs:1435-1437) of each CompressedEdwardsY: a list of bool."""
        return [bool(f & 2) for f in _torsion_flags(points, engine)]

    @staticmethod
    def hash_to_curve_batch(messages, dst, engine=None):
        """EdwardsPoint::hash_to_curve::<Sha512> (edwards.rs:736-750, RFC 9380 edwards25519_XMD:SHA-512_ELL2_RO_) for each
        message, with one domain separation tag of 1..255 bytes: the list of 32-byte CompressedEdwardsY encodings."""
        eng = engine or default_engine()
        flat, offs, n = _flat_messages(messages)
        raw = eng.edwards_hash_to_curve_batch(flat, offs, n, dst)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    @staticmethod
    def encode_to_curve_batch(messages, dst, engine=None):
        """EdwardsPoint::encode_to_curve::<Sha512> (edwards.rs:710-721, ..._ELL2_NU_), like hash_to_curve_batch."""
        eng = engine or default_engine()
        flat, offs, n = _flat_messages(messages)
        raw = eng.edwards_encode_to_curve_batch(flat, offs, n, dst)
        return [raw[32 * i:32 * i + 32] for i in range(n)]


def _mul_batch(scalars, points, fmt, clamped, engine):
    single_s, ss = _items(scalars, 32, "scalars")
    single_p, ps = _items(points, 32, "points")
    if not single_s and not single_p and len(ss) != len(ps):
        raise ValueError("scalars and points must have the same length (or one of them be a single item)")
    n = len(ps) if single_s else len(ss)
    if n == 0:
        return []
    if not clamped and any(s[31] & 0x80 for s in ss):
        raise ValueError("a scalar has bit 255 set")
    eng = engine or default_engine()
    rc, raw, _ = eng.mul_batch(b"".join(ss), len(ss), b"".join(ps), len(ps), n, fmt, clamped=clamped)
    if rc == 1:
        raise ValueError("a point does not decode")
    outs = [raw[32 * i:32 * i + 32] for i in range(n)]
    return outs[0] if single_s and single_p else outs


def _mul_base_batch(scalars, fmt, clamped, engine):
    single, ss = _items(scalars, 32, "scalars")
    if not ss:
        return []
    if not clamped and any(s[31] & 0x80 for s in ss):
        raise ValueError("a scalar has bit 255 set")
    eng = engine or default_engine()
    raw = eng.mul_base_ct_batch(b"".join(ss), len(ss), fmt, clamped=clamped)
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ss))]
    return outs[0] if single else outs


def _scalar_binary(a, b, op, engine):
    single_a, as_ = _items(a, 32, "scalars")
    single_b, bs = _items(b, 32, "scalars")
    n = _broadcast_len(single_a, as_, single_b, bs)
    if n == 0:
        return []
    eng = engine or default_engine()
    raw = eng.scalar_binary_batch(op, b"".join(as_), len(as_), b"".join(bs), len(bs), n)
    outs = [raw[32 * i:32 * i + 32] for i in range(n)]
    return outs[0] if single_a and single_b else outs


def _scalar_unary(scalars, op, engine):
    single, ss = _items(scalars, 32, "scalars")
    if not ss:
        return []
    eng = engine or default_engine()
    raw = eng.scalar_unary_batch(op, b"".join(ss), len(ss))
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ss))]
    return outs[0] if single else outs


def _scalar_fold_batch(scalar_lists, op, engine):
    import array
    lists = [_items(list(s), 32, "scalars")[1] for s in scalar_lists]
    m = len(lists)
    if m == 0:
        return []
    offs = array.array("Q", [0])
    for s in lists:
        offs.append(offs[-1] + len(s))
    eng = engine or default_engine()
    raw = eng.scalar_fold_batch(op, b"".join(b"".join(s) for s in lists) or b"\0", offs.tobytes(), m)
    return [raw[32 * j:32 * j + 32] for j in range(m)]


class Scalar:
    """Mirror of curve25519_dalek::scalar::Scalar (scalar.rs) on 32-byte little-endian encodings, batched on the GPU.  One
    item (bytes) gives one result, a list gives the list; in the binary forms a single item is used for every item of the
    other operand.  The arithmetic takes canonical scalars (< l, invariant #2) and returns canonical ones; a
    non-canonical input raises EngineError (the reference's Add and Sub are wrong for unreduced scalars, so nothing is
    reduced silently).  Constant time in the scalar values."""

    @staticmethod
    def from_bytes_mod_order_batch(data, engine=None):
        """Scalar::from_bytes_mod_order (scalar.rs:235-244): any 32 bytes, reduced mod l."""
        single, items = _items(data, 32, "scalar encodings")
        if not items:
            return []
        eng = engine or default_engine()
        _, raw, _ = eng.scalar_from_bytes_batch(b"".join(items), len(items))
        outs = [raw[32 * i:32 * i + 32] for i in range(len(items))]
        return outs[0] if single else outs

    @staticmethod
    def from_bytes_mod_order_wide_batch(data, engine=None):
        """Scalar::from_bytes_mod_order_wide (scalar.rs:248-250): any 64 bytes, reduced mod l."""
        single, items = _items(data, 64, "wide scalar encodings")
        if not items:
            return []
        eng = engine or default_engine()
        raw = eng.scalar_from_wide_batch(b"".join(items), len(items))
        outs = [raw[32 * i:32 * i + 32] for i in range(len(items))]
        return outs[0] if single else outs

    @staticmethod
    def from_canonical_bytes_batch(data, engine=None):
        """Scalar::from_canonical_bytes (scalar.rs:259-263): the 32 bytes when canonical, else None."""
        single, items = _items(data, 32, "scalar encodings")
        if not items:
            return []
        eng = engine or default_engine()
        _, raw, ok = eng.scalar_from_bytes_batch(b"".join(items), len(items), canonical=True)
        outs = [raw[32 * i:32 * i + 32] if ok[i] else None for i in range(len(items))]
        return outs[0] if single else outs

    @staticmethod
    def hash_from_bytes_batch(messages, engine=None):
        """Scalar::hash_from_bytes::<Sha512> (scalar.rs:617-624): SHA-512 of each message mod l, the list of scalars."""
        eng = engine or default_engine()
        flat, offs, n = _flat_messages(messages)
        raw = eng.scalar_hash_from_bytes_batch(flat, offs, n)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    @staticmethod
    def add_batch(a, b, engine=None):
        """Add (scalar.rs:334-349): a + b mod l."""
        return _scalar_binary(a, b, "add", engine)

    @staticmethod
    def sub_batch(a, b, engine=None):
        """Sub (scalar.rs:354-362): a - b mod l."""
        return _scalar_binary(a, b, "sub", engine)

    @staticmethod
    def mul_batch(a, b, engine=None):
        """Mul (scalar.rs:317-322): a b mod l."""
        return _scalar_binary(a, b, "mul", engine)

    @staticmethod
    def neg_batch(scalars, engine=None):
        """Neg (scalar.rs:366-374): -s mod l (0 for 0)."""
        return _scalar_unary(scalars, "neg", engine)

    @staticmethod
    def div_by_2_batch(scalars, engine=None):
        """Scalar::div_by_2 (scalar.rs:858-870): s / 2 mod l."""
        return _scalar_unary(scalars, "div_by_2", engine)

    @staticmethod
    def invert_each(scalars, engine=None):
        """Scalar::invert (scalar.rs:739-741) of each scalar on its own: s^(l-2), so 0 gives 0.  Not the reference's
        invert_batch, which requires nonzero inputs and returns the product of the inverses."""
        return _scalar_unary(scalars, "invert", engine)

    @staticmethod
    def invert_batch_alloc(scalars, engine=None):
        """Scalar::invert_batch_alloc (scalar.rs:802-853): (the list of inverses, the product of all inverses).  Inputs are
        taken mod l; a zero input raises EngineError, as the reference requires nonzero inputs."""
        _, ss = _items(list(scalars), 32, "scalars")
        eng = engine or default_engine()
        raw, prod = eng.scalar_invert_batch(b"".join(ss) or b"\0", len(ss))
        return [raw[32 * i:32 * i + 32] for i in range(len(ss))], prod

    @staticmethod
    def sum(scalars, engine=None):
        """Sum<T> (scalar.rs:466-476): the sum of the scalars, 0 when there are none."""
        return _scalar_fold_batch([list(scalars)], "sum", engine)[0]

    @staticmethod
    def sum_batch(scalar_lists, engine=None):
        """The Sum of each list of scalars, one call for all lists."""
        return _scalar_fold_batch(scalar_lists, "sum", engine)

    @staticmethod
    def product(scalars, engine=None):
        """Product<T> (scalar.rs:454-464): the product of the scalars, 1 when there are none."""
        return _scalar_fold_batch([list(scalars)], "product", engine)[0]

    @staticmethod
    def product_batch(scalar_lists, engine=None):
        """The Product of each list of scalars, one call for all lists."""
        return _scalar_fold_batch(scalar_lists, "product", engine)


class MontgomeryPoint:
    """Mirror of curve25519_dalek::montgomery::MontgomeryPoint (montgomery.rs).  Points are their 32-byte u coordinates,
    read like FieldElement::from_bytes (bit 255 ignored, values in [p, 2^255) accepted, twist points accepted); results
    are canonical.  One item gives one result, a list gives the list; a single scalar or point is used for every item."""

    @staticmethod
    def mul_batch(scalars, points, engine=None):
        """Scalar * MontgomeryPoint (montgomery.rs:484-505): u([s] P) for 32-byte scalars with bit 255 clear (not clamped,
        not reduced), constant time."""
        single_s, ss = _items(scalars, 32, "scalars")
        single_p, ps = _items(points, 32, "points")
        n = _broadcast_len(single_s, ss, single_p, ps)
        if n == 0:
            return []
        if any(s[31] & 0x80 for s in ss):
            raise ValueError("a scalar has bit 255 set")
        eng = engine or default_engine()
        raw = eng.montgomery_mul_batch(b"".join(ss), len(ss), b"".join(ps), len(ps), n)
        outs = [raw[32 * i:32 * i + 32] for i in range(n)]
        return outs[0] if single_s and single_p else outs

    @staticmethod
    def mul_bits_be_batch(ints, nbits, points, engine=None):
        """MontgomeryPoint::mul_bits_be (montgomery.rs:176-211) over bits nbits-1..0 of little-endian integers of one
        common length of 1..64 bytes (nbits <= 8 x that length), constant time in the bits."""
        single_i = isinstance(ints, (bytes, bytearray))
        items = [bytes(ints)] if single_i else [bytes(x) for x in ints]
        int_bytes = len(items[0]) if items else 1
        if any(len(x) != int_bytes for x in items) or not 1 <= int_bytes <= 64:
            raise ValueError("the integers are 1..64 bytes each, all of one length")
        if not 0 <= nbits <= 8 * int_bytes:
            raise ValueError("nbits must be between 0 and 8 x the integers' length")
        single_p, ps = _items(points, 32, "points")
        n = _broadcast_len(single_i, items, single_p, ps)
        if n == 0:
            return []
        eng = engine or default_engine()
        raw = eng.montgomery_mul_bits_be_batch(b"".join(items), int_bytes, len(items), nbits, b"".join(ps), len(ps), n)
        outs = [raw[32 * i:32 * i + 32] for i in range(n)]
        return outs[0] if single_i and single_p else outs

    @staticmethod
    def to_edwards_batch(points, signs, engine=None):
        """MontgomeryPoint::to_edwards (montgomery.rs:223-268) for each u coordinate with its sign (a u8: only bit 0
        counts; one int is used for every item): the CompressedEdwardsY of the point, or None for u = -1 and for u of the
        twist.  Returns a list."""
        _, ps = _items(points, 32, "points")
        sg = [signs] * len(ps) if isinstance(signs, int) else [int(x) for x in signs]
        if len(sg) != len(ps):
            raise ValueError("one sign per point")
        if any(not 0 <= x <= 255 for x in sg):
            raise ValueError("signs are u8 values")
        if not ps:
            return []
        eng = engine or default_engine()
        _, raw, ok = eng.montgomery_to_edwards_batch(b"".join(ps), bytes(sg), len(ps))
        return [raw[32 * i:32 * i + 32] if ok[i] else None for i in range(len(ps))]

    @staticmethod
    def mul_base_batch(scalars, engine=None):
        """MontgomeryPoint::mul_base (montgomery.rs:143-146): u(s B) for 32-byte scalars with bit 255 clear, constant time."""
        return _mul_base_batch(scalars, POINTS_MONTGOMERY, False, engine)

    @staticmethod
    def mul_clamped_batch(bytes_list, points, engine=None):
        """MontgomeryPoint::mul_clamped (montgomery.rs:150-161): x25519(bytes, u), through the X25519 batch."""
        single_s, ss = _items(bytes_list, 32, "scalars")
        single_p, ps = _items(points, 32, "points")
        n = _broadcast_len(single_s, ss, single_p, ps)
        if n == 0:
            return []
        outs = x25519(ss * n if len(ss) == 1 else ss, ps * n if len(ps) == 1 else ps, engine=engine)
        return outs[0] if single_s and single_p else outs

    @staticmethod
    def mul_base_clamped_batch(bytes_list, engine=None):
        """MontgomeryPoint::mul_base_clamped (montgomery.rs:164-174): the X25519 public key of each 32-byte secret."""
        single, ss = _items(bytes_list, 32, "scalars")
        if not ss:
            return []
        outs = x25519_public_keys(ss, engine=engine)
        return outs[0] if single else outs


def _broadcast_len(single_a, a, single_b, b):
    if not single_a and not single_b and len(a) != len(b):
        raise ValueError("the inputs must have the same length (or one of them be a single item)")
    return len(b) if single_a else len(a)


def _double_base_batch(a_list, points, b_list, fmt, engine):
    _, as_ = _items(a_list, 32, "scalars")
    _, bs = _items(b_list, 32, "scalars")
    _, ps = _items(points, 32, "points")
    if not len(as_) == len(bs) == len(ps):
        raise ValueError("a_list, points and b_list must have the same length")
    n = len(ps)
    if n == 0:
        return []
    if any((a[31] | b[31]) & 0x80 for a, b in zip(as_, bs)):
        raise ValueError("a scalar has bit 255 set")
    eng = engine or default_engine()
    rc, raw, _ = eng.vartime_double_base_batch(b"".join(a + b for a, b in zip(as_, bs)), b"".join(ps), n, fmt)
    if rc == 1:
        raise ValueError("a point does not decode")
    return [raw[32 * i:32 * i + 32] for i in range(n)]


def _torsion_flags(points, engine):
    _, ps = _items(points, 32, "points")
    if not ps:
        return []
    eng = engine or default_engine()
    flags = eng.torsion_batch(b"".join(ps), len(ps))
    if any(f == 0 for f in flags):
        raise ValueError("a point does not decode")
    return flags


def _flat_messages(messages):
    """Messages back to back with n + 1 u64 offsets (the layout of verify_batch_flat); the buffer is never empty."""
    msgs = [bytes(m) for m in messages]
    n = len(msgs)
    offs = (C.c_uint64 * (n + 1))()
    acc = 0
    for i, m in enumerate(msgs):
        offs[i] = acc
        acc += len(m)
    offs[n] = acc
    flat = b"".join(msgs) + b"\0"
    return flat, offs, n


X25519_BASEPOINT_BYTES = bytes([9]) + bytes(31)      # x25519-dalek x25519.rs:385, u = 9


def _x25519_items(xs):
    single = isinstance(xs, (bytes, bytearray))
    items = [bytes(xs)] if single else [bytes(x) for x in xs]
    if any(len(x) != 32 for x in items):
        raise ValueError("X25519 secrets and u coordinates are 32 bytes each")
    return single, items


def x25519(scalars, us, engine=None):
    """x25519-dalek's x25519(k, u) (x25519.rs:390-392).  One 32-byte secret and u coordinate give 32 bytes; lists of
    them give the list of shared secrets, computed in one batch."""
    single, ks = _x25519_items(scalars)
    _, vs = _x25519_items(us)
    if len(ks) != len(vs):
        raise ValueError("scalars and us must have the same length")
    eng = engine or default_engine()
    raw, _ = eng.x25519_batch(b"".join(ks), b"".join(vs), len(ks))
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ks))]
    return outs[0] if single else outs


def x25519_public_keys(secrets, engine=None):
    """PublicKey::from(&StaticSecret) (x25519.rs:105-110) for each 32-byte secret: one secret gives its 32-byte public
    key, a list gives the list."""
    single, ks = _x25519_items(secrets)
    eng = engine or default_engine()
    raw = eng.x25519_public_keys(b"".join(ks), len(ks))
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ks))]
    return outs[0] if single else outs


def _items(xs, size, what):
    single = isinstance(xs, (bytes, bytearray))
    items = [bytes(xs)] if single else [bytes(x) for x in xs]
    if any(len(x) != size for x in items):
        raise ValueError("%s are %d bytes each" % (what, size))
    return single, items


def ed25519_verifying_keys(seeds, engine=None):
    """SigningKey::from_bytes(seed).verifying_key() (signing.rs:106, :171) for each 32-byte seed: one seed gives its
    32-byte VerifyingKey, a list gives the list."""
    single, ks = _items(seeds, 32, "Ed25519 seeds")
    eng = engine or default_engine()
    raw = eng.verifying_keys(b"".join(ks), len(ks))
    outs = [raw[32 * i:32 * i + 32] for i in range(len(ks))]
    return outs[0] if single else outs


def ed25519_to_montgomery(verifying_keys, engine=None):
    """VerifyingKey::to_montgomery (ed25519-dalek verifying.rs:476): the Montgomery u of each 32-byte verifying key, None
    for a key that does not decompress.  One key gives one result, a list gives the list."""
    single, ks = _items(verifying_keys, 32, "verifying keys")
    if not ks:
        return []
    eng = engine or default_engine()
    _, limbs, ok = eng.decompress_batch(b"".join(ks), len(ks))
    raw = eng.edwards_to_montgomery_batch(limbs, len(ks))
    outs = [raw[32 * i:32 * i + 32] if ok[i] else None for i in range(len(ks))]
    return outs[0] if single else outs


def _sign_args(seeds, n):
    single_key, ks = _items(seeds, 32, "Ed25519 seeds")
    if not single_key and len(ks) not in (1, n):
        raise ValueError("one seed, or one seed per message")
    return ks


def ed25519_sign(seeds, messages, engine=None):
    """Signer::sign (signing.rs:566-571) on the GPU.  `messages` is one message (bytes) or a list; `seeds` is one 32-byte
    seed, which signs every message, or a list with one seed per message.  Returns the 64-byte signature, or the list."""
    single = isinstance(messages, (bytes, bytearray))
    msgs = [bytes(messages)] if single else [bytes(m) for m in messages]
    ks = _sign_args(seeds, len(msgs))
    eng = engine or default_engine()
    flat, offs, n = _flat_messages(msgs)
    raw = eng.sign_flat(b"".join(ks), len(ks) if n else 0, flat, offs, n) if n else b""
    outs = [raw[64 * i:64 * i + 64] for i in range(n)]
    return outs[0] if single else outs


def _prehash_items(prehashed):
    """64-byte digests, or objects with .digest() such as hashlib.sha512 (the reference's MsgDigest)."""
    single = isinstance(prehashed, (bytes, bytearray)) or hasattr(prehashed, "digest")
    items = [prehashed] if single else list(prehashed)
    out = [bytes(p.digest()) if hasattr(p, "digest") else bytes(p) for p in items]
    if any(len(p) != 64 for p in out):
        raise ValueError("Ed25519ph prehashes are 64-byte digests")
    return single, out


def ed25519_sign_prehashed(seeds, prehashed, context=None, engine=None):
    """SigningKey::sign_prehashed (signing.rs:312, Ed25519ph) on the GPU.  `prehashed` is one digest or a list (64 bytes
    each, or objects with .digest() such as hashlib.sha512(message)); `seeds` as in ed25519_sign.  Raises
    SignatureError(5) (PrehashedContextLength) for a context longer than 255 bytes."""
    single, phs = _prehash_items(prehashed)
    ks = _sign_args(seeds, len(phs))
    eng = engine or default_engine()
    n = len(phs)
    rc, raw = eng.sign_prehashed(b"".join(ks), len(ks) if n else 0, b"".join(phs), n, context)
    if rc:
        raise SignatureError(rc)
    outs = [raw[64 * i:64 * i + 64] for i in range(n)]
    return outs[0] if single else outs


def _raw_sign_args(esks, vks, n):
    single_e, es = _items(esks, 64, "ExpandedSecretKey bytes")
    single_v, vs = _items(vks, 32, "verifying keys")
    if len(es) != len(vs) or single_e != single_v:
        raise ValueError("one verifying key per ExpandedSecretKey")
    if not single_e and len(es) not in (1, n):
        raise ValueError("one key, or one key per message")
    return es, vs


def ed25519_expanded_verifying_keys(esks, engine=None):
    """VerifyingKey::from(&ExpandedSecretKey::from_bytes(esk)) (hazmat.rs:84-99, verifying.rs:97-102) for each 64-byte
    ExpandedSecretKey (scalar bytes, then hash_prefix): one gives its 32-byte VerifyingKey, a list gives the list."""
    single, es = _items(esks, 64, "ExpandedSecretKey bytes")
    eng = engine or default_engine()
    raw = eng.expanded_verifying_keys(b"".join(es), len(es))
    outs = [raw[32 * i:32 * i + 32] for i in range(len(es))]
    return outs[0] if single else outs


def ed25519_raw_sign(esks, messages, verifying_keys, engine=None):
    """hazmat::raw_sign::<Sha512> (hazmat.rs:137) on the GPU.  `messages` is one message or a list; `esks` is one 64-byte
    ExpandedSecretKey, which signs every message, or one per message, and `verifying_keys` matches it.  The verifying keys
    are hashed as given and not decoded: the caller makes sure they decode, as the reference's VerifyingKey type does."""
    single = isinstance(messages, (bytes, bytearray))
    msgs = [bytes(messages)] if single else [bytes(m) for m in messages]
    es, vs = _raw_sign_args(esks, verifying_keys, len(msgs))
    eng = engine or default_engine()
    flat, offs, n = _flat_messages(msgs)
    raw = eng.raw_sign_flat(b"".join(es), b"".join(vs), len(es), flat, offs, n) if n else b""
    outs = [raw[64 * i:64 * i + 64] for i in range(n)]
    return outs[0] if single else outs


def ed25519_raw_sign_prehashed(esks, prehashed, verifying_keys, context=None, engine=None):
    """hazmat::raw_sign_prehashed::<Sha512, Sha512> (hazmat.rs:182, Ed25519ph) on the GPU; `prehashed` as in
    ed25519_sign_prehashed, keys as in ed25519_raw_sign.  Raises SignatureError(5) for a context longer than 255 bytes."""
    single, phs = _prehash_items(prehashed)
    es, vs = _raw_sign_args(esks, verifying_keys, len(phs))
    eng = engine or default_engine()
    n = len(phs)
    rc, raw = eng.raw_sign_prehashed(b"".join(es), b"".join(vs), len(es) if n else 0, b"".join(phs), n, context)
    if rc:
        raise SignatureError(rc)
    outs = [raw[64 * i:64 * i + 64] for i in range(n)]
    return outs[0] if single else outs


def ed25519_verify_prehashed(prehashed, signatures, verifying_keys, context=None, strict=False, engine=None):
    """VerifyingKey::verify_prehashed / verify_prehashed_strict (verifying.rs:230-257, :424-459) of each signature: the
    list of result codes (0 Ok, 1 Verify, 3 ScalarFormat, 4 PointDecompression), or one code for a single item.  A
    context longer than 255 bytes raises ValueError."""
    single, phs = _prehash_items(prehashed)
    _, sigs = _items([signatures] if single else signatures, 64, "signatures")
    _, keys = _items([verifying_keys] if single else verifying_keys, 32, "verifying keys")
    if not (len(phs) == len(sigs) == len(keys)):
        raise ValueError("prehashes, signatures and verifying keys must have the same length")
    if context is not None and len(bytes(context)) > 255:
        raise ValueError("an Ed25519ph context is at most 255 bytes")
    eng = engine or default_engine()
    _, res = eng.verify_prehashed_each(b"".join(phs), b"".join(sigs), b"".join(keys), len(phs), context, strict)
    return res[0] if single else res


class _Precomputation:
    """VartimePrecomputedMultiscalarMul (traits.rs:290-406): static points converted once, resident on the GPU."""
    _FMT = POINTS_COMPRESSED

    def __init__(self, static_points, engine=None, fmt=None):
        """`new` (traits.rs:297-300): static_points = iterable of 32-byte encodings (or, with fmt=POINTS_EXTENDED, a
        buffer of n x 20 u64 limbs passed as (buffer, n))."""
        self.eng = engine or default_engine()
        fmt = self._FMT if fmt is None else fmt
        if fmt == POINTS_EXTENDED:
            buf, n = static_points
        else:
            pts = list(static_points)
            buf, n = b"".join(pts), len(pts)
        h = C.c_void_p()
        rc = self.eng._check(self.eng.lib.dalek_b200_precomp_new(self.eng.h, _ptr(buf) if n else None, fmt, n, C.byref(h)))
        if rc == 1:
            raise ValueError("a static point does not decode")
        self.h = h

    def __len__(self):                                   # traits.rs:303
        return int(self.eng.lib.dalek_b200_precomp_len(self.h))

    def is_empty(self):                                  # traits.rs:306
        return len(self) == 0

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.dalek_b200_precomp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def optional_mixed_multiscalar_mul(self, static_scalars, dynamic_scalars, dynamic_points, dynamic_fmt=None):
        """traits.rs:402-413.  A dynamic point that is None or undecodable gives None."""
        ss, ds, dp = list(static_scalars), list(dynamic_scalars), list(dynamic_points)
        assert len(ss) <= len(self), "more static scalars than static points"
        assert len(ds) == len(dp), "dynamic scalars and points must have the same length"
        if any(p is None for p in dp):
            return None
        out = (C.c_uint8 * 32)()
        sb, db, pb = b"".join(ss), b"".join(ds), b"".join(dp)      # kept alive across the call
        rc = self.eng._check(self.eng.lib.dalek_b200_precomp_mixed_msm(
            self.eng.h, self.h, _ptr(sb) if ss else None, len(ss), _ptr(db) if ds else None, _ptr(pb) if dp else None,
            self._FMT if dynamic_fmt is None else dynamic_fmt, len(ds), C.addressof(out), None))
        return None if rc == 1 else bytes(out)

    def vartime_mixed_multiscalar_mul(self, static_scalars, dynamic_scalars, dynamic_points):
        """traits.rs:357-383: .expect() on the optional form."""
        r = self.optional_mixed_multiscalar_mul(static_scalars, dynamic_scalars, dynamic_points)
        if r is None:
            raise ValueError("should return some point")
        return r

    def vartime_multiscalar_mul(self, static_scalars):
        """traits.rs:324-338."""
        return self.vartime_mixed_multiscalar_mul(static_scalars, [], [])


class VartimeEdwardsPrecomputation(_Precomputation):
    """curve25519-dalek/src/edwards.rs:1038-1076 (CompressedEdwardsY encodings in and out)."""
    _FMT = POINTS_COMPRESSED


class VartimeRistrettoPrecomputation(_Precomputation):
    """curve25519-dalek/src/ristretto.rs:1004-1049 (CompressedRistretto encodings in and out)."""
    _FMT = POINTS_RISTRETTO


class _BasepointTable:
    """BasepointTable (traits.rs:50-74) for k >= 1 points at once, resident on the GPU: the comb tables of every point
    stay in device memory until close(), and each multiplication sends scalars (and table indices) only."""
    _FMT = POINTS_COMPRESSED

    def __init__(self, points, engine=None, fmt=None):
        """points = iterable of 32-byte encodings (or, with fmt=POINTS_EXTENDED, a buffer of k x 20 u64 limbs passed as
        (buffer, k)).  A point that does not decode raises ValueError naming the first one."""
        self.h = None
        self.eng = engine or default_engine()
        fmt = self._FMT if fmt is None else fmt
        if fmt == POINTS_EXTENDED:
            if self._FMT == POINTS_RISTRETTO:
                raise ValueError("Ristretto tables are made from CompressedRistretto encodings")
            buf, k = points
            nbytes = buf.nbytes if hasattr(buf, "nbytes") else (buf.numel() * buf.element_size() if hasattr(buf, "numel")
                                                                else len(buf))
            if nbytes < 160 * k:
                raise ValueError("%d extended points take %d bytes, the buffer holds %d" % (k, 160 * k, nbytes))
        else:
            _, pts = _items(list(points), 32, "points")
            buf, k = b"".join(pts), len(pts)
        if k == 0:
            raise ValueError("a basepoint table needs at least one point")
        rc, h, ok = self.eng.basepoint_tables_new(buf, k, fmt)
        if rc == 1:
            raise ValueError("point %d does not decode" % ok.index(0))
        self.h, self.k, self._bases = h, k, None

    @classmethod
    def create(cls, point, engine=None):
        """create (traits.rs:56): the table of one point."""
        return cls([point], engine=engine)

    def __len__(self):
        return self.k

    def basepoint(self, i=0):
        """basepoint (traits.rs:59): the canonical encoding of point i, read back from its table (all k once, then kept)."""
        if not 0 <= i < self.k:
            raise IndexError("table index out of range")
        if self._bases is None:
            self._bases = self.eng.basepoint_tables_basepoints(self.h)
        return self._bases[32 * i:32 * i + 32]

    def _mul(self, scalars, indices, clamped):
        single, ss = _items(scalars, 32, "scalars")
        if not ss:
            return []
        if not clamped and any(s[31] & 0x80 for s in ss):
            raise ValueError("a scalar has bit 255 set")
        idx = None
        if indices is not None:
            import array
            idx = array.array("I", indices)
            if len(idx) != len(ss):
                raise ValueError("one table index per scalar")
            if max(idx) >= self.k:
                raise ValueError("a table index is not below len()")
            idx = idx.tobytes()
        raw = self.eng.basepoint_tables_mul(self.h, b"".join(ss), idx, len(ss), clamped=clamped)
        outs = [raw[32 * i:32 * i + 32] for i in range(len(ss))]
        return outs[0] if single else outs

    def mul_base_batch(self, scalars, indices=None):
        """mul_base (traits.rs:62) for each 32-byte scalar (bit 255 clear, not reduced), through table indices[i] (None:
        table 0).  Constant time in the scalars.  Returns the encoding, or the list."""
        return self._mul(scalars, indices, False)

    def mul_base_clamped_batch(self, bytes_list, indices=None):
        """mul_base_clamped (traits.rs:66-74): any 32 bytes, clamped and not reduced; like mul_base_batch."""
        return self._mul(bytes_list, indices, True)

    def close(self):
        if getattr(self, "h", None):
            self.eng.basepoint_tables_destroy(self.h)          # does not use the engine's context: safe after its close()
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class EdwardsBasepointTable(_BasepointTable):
    """EdwardsBasepointTable (edwards.rs:1127-1243): CompressedEdwardsY (or extended limbs) in, CompressedEdwardsY out."""
    _FMT = POINTS_COMPRESSED


class RistrettoBasepointTable(_BasepointTable):
    """RistrettoBasepointTable (ristretto.rs:1080-1115): CompressedRistretto in and out."""
    _FMT = POINTS_RISTRETTO


class VerifyingKeySet:
    """k VerifyingKeys (VerifyingKey::from_bytes, verifying.rs:167-175) resident on the GPU: each key is decompressed and
    tabulated once, and every later call sends messages, signatures and key indices only."""

    def __init__(self, verifying_keys, engine=None):
        """verifying_keys = iterable of 32-byte encodings, kept as given (the challenge hashes them).  A key that does not
        decode raises SignatureError (PointDecompression) naming the first one."""
        self.h = None
        self.eng = engine or default_engine()
        _, keys = _items(list(verifying_keys), 32, "verifying keys")
        if not keys:
            raise ValueError("a verifying-key set needs at least one key")
        rc, h, ok, weak = self.eng.key_set_new(b"".join(keys), len(keys))
        if rc:
            err = SignatureError(rc)
            err.args = ("%s: verifying key %d does not decode" % (err.kind, ok.index(0)),)
            raise err
        self.h, self.k, self._weak = h, len(keys), weak

    def __len__(self):
        return self.k

    def is_weak(self, i=0):
        """VerifyingKey::is_weak (verifying.rs:192-194) of key i: a key of small order."""
        if not 0 <= i < self.k:
            raise IndexError("key index out of range")
        return bool(self._weak[i])

    def _indices(self, indices, n):
        if indices is None:
            return None
        import array
        idx = array.array("I", indices)
        if len(idx) != n:
            raise ValueError("one key index per signature")
        if n and max(idx) >= self.k:
            raise ValueError("a key index is not below len()")
        return idx.tobytes()

    def verify_each(self, messages, signatures, indices=None, strict=False):
        """VerifyingKey::verify / verify_strict (verifying.rs:203-219, :359-382) of signature i over message i under key
        indices[i] (None: key 0): the list of result codes (0 Ok, 1 Verify, 3 ScalarFormat), or one code for a single
        message."""
        single = isinstance(messages, (bytes, bytearray))
        msgs = [bytes(messages)] if single else [bytes(m) for m in messages]
        _, sigs = _items([signatures] if single else signatures, 64, "signatures")
        if len(sigs) != len(msgs):
            raise ValueError("messages and signatures must have the same length")
        idx = self._indices([indices] if single and indices is not None else indices, len(msgs))
        flat, offs, n = _flat_messages(msgs)
        _, res = self.eng.key_set_verify_flat(self.h, flat, offs, b"".join(sigs), idx, n, strict)
        return res[0] if single else res

    def verify_prehashed_each(self, prehashed, signatures, indices=None, context=None, strict=False):
        """VerifyingKey::verify_prehashed / verify_prehashed_strict (verifying.rs:230-257, :424-459) of each signature
        under key indices[i], as ed25519_verify_prehashed.  A context longer than 255 bytes raises ValueError."""
        single, phs = _prehash_items(prehashed)
        _, sigs = _items([signatures] if single else signatures, 64, "signatures")
        if len(sigs) != len(phs):
            raise ValueError("prehashes and signatures must have the same length")
        if context is not None and len(bytes(context)) > 255:
            raise ValueError("an Ed25519ph context is at most 255 bytes")
        idx = self._indices([indices] if single and indices is not None else indices, len(phs))
        _, res = self.eng.key_set_verify_prehashed(self.h, b"".join(phs), b"".join(sigs), idx, len(phs), context, strict)
        return res[0] if single else res

    def close(self):
        if getattr(self, "h", None):
            self.eng.key_set_destroy(self.h)                   # does not use the engine's context: safe after its close()
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


SIGNING_KEY_SEED, SIGNING_KEY_KEYPAIR, SIGNING_KEY_EXPANDED = 0, 1, 2        # DALEK_SIGNING_KEY_*


class SigningKeySet:
    """k Ed25519 signing keys resident on the GPU: each key is derived once (its clamped scalar, hash_prefix and
    verifying key stay in device memory until close(), which clears them), and every later call sends messages and key
    indices only.  Make one with from_seeds, from_keypair_bytes or from_expanded."""

    def __init__(self, keys, form, engine=None):
        self.h = None
        self.eng = engine or default_engine()
        size = 32 if form == SIGNING_KEY_SEED else 64
        _, ks = _items(list(keys), size, "keys of this form")
        if not ks:
            raise ValueError("a signing-key set needs at least one key")
        rc, h, status = self.eng.signing_key_set_new(b"".join(ks), len(ks), form)
        if rc:
            err = SignatureError(rc)
            err.args = ("%s: key %d" % (err.kind, next(i for i, c in enumerate(status) if c)),)
            raise err
        self.h, self.k, self._pks = h, len(ks), None

    @classmethod
    def from_seeds(cls, seeds, engine=None):
        """SigningKey::from_bytes (signing.rs:106) for each 32-byte seed."""
        return cls(seeds, SIGNING_KEY_SEED, engine)

    @classmethod
    def from_keypair_bytes(cls, keypairs, engine=None):
        """SigningKey::from_keypair_bytes (signing.rs:140-150) for each 64-byte seed || verifying key.  Raises
        SignatureError naming the first key whose public half does not decode (PointDecompression) or is not the key
        derived from the seed, byte for byte (MismatchedKeypair)."""
        return cls(keypairs, SIGNING_KEY_KEYPAIR, engine)

    @classmethod
    def from_expanded(cls, esks, engine=None):
        """ExpandedSecretKey::from_bytes (hazmat.rs:84-99) for each 64 bytes (scalar bytes, then hash_prefix), with the
        verifying key derived from it."""
        return cls(esks, SIGNING_KEY_EXPANDED, engine)

    def __len__(self):
        return self.k

    def verifying_keys(self):
        """The 32-byte VerifyingKey of every key, in order."""
        if self._pks is None:
            raw = self.eng.signing_key_set_verifying_keys(self.h)
            self._pks = [raw[32 * i:32 * i + 32] for i in range(self.k)]
        return list(self._pks)

    def verifying_key(self, i=0):
        """SigningKey::verifying_key (signing.rs:171) of key i."""
        if not 0 <= i < self.k:
            raise IndexError("key index out of range")
        return self.verifying_keys()[i]

    def _indices(self, indices, n):
        if indices is None:
            return None
        import array
        idx = array.array("I", indices)
        if len(idx) != n:
            raise ValueError("one key index per message")
        if n and max(idx) >= self.k:
            raise ValueError("a key index is not below len()")
        return idx.tobytes()

    def sign(self, messages, indices=None):
        """Signer::sign (signing.rs:566-571) of message i under key indices[i] (None: key 0).  One message (bytes) and
        one index give one 64-byte signature; lists give the list."""
        single = isinstance(messages, (bytes, bytearray))
        msgs = [bytes(messages)] if single else [bytes(m) for m in messages]
        idx = self._indices([indices] if single and indices is not None else indices, len(msgs))
        flat, offs, n = _flat_messages(msgs)
        raw = self.eng.signing_key_set_sign_flat(self.h, flat, offs, idx, n) if n else b""
        outs = [raw[64 * i:64 * i + 64] for i in range(n)]
        return outs[0] if single else outs

    def sign_prehashed(self, prehashed, indices=None, context=None):
        """SigningKey::sign_prehashed (signing.rs:312, Ed25519ph) of each prehash under key indices[i], as
        ed25519_sign_prehashed.  Raises SignatureError(5) for a context longer than 255 bytes."""
        single, phs = _prehash_items(prehashed)
        idx = self._indices([indices] if single and indices is not None else indices, len(phs))
        n = len(phs)
        rc, raw = self.eng.signing_key_set_sign_prehashed(self.h, b"".join(phs), idx, n, context)
        if rc:
            raise SignatureError(rc)
        outs = [raw[64 * i:64 * i + 64] for i in range(n)]
        return outs[0] if single else outs

    def close(self):
        if getattr(self, "h", None):
            self.eng.signing_key_set_destroy(self.h)           # does not use the engine's context: safe after its close()
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RistrettoPoint(_GroupOps):
    """Mirror of the forwarding impls in curve25519-dalek/src/ristretto.rs:964-994 (CompressedRistretto I/O)."""
    _FMT = POINTS_RISTRETTO

    @staticmethod
    def vartime_multiscalar_mul(scalars, points, engine=None):
        scalars, points = list(scalars), list(points)
        assert len(scalars) == len(points)
        eng = engine or default_engine()
        rc, comp = eng.ristretto_vartime_msm(b"".join(scalars), b"".join(points), len(scalars))
        if rc == 1:
            raise ValueError("should return some point")
        return comp

    @staticmethod
    def optional_multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        """optional_multiscalar_mul (ristretto.rs:979-994) for many independent MSMs in one call over CompressedRistretto
        points: the list of CompressedRistretto results, None where a point is None or does not decode."""
        return _msm_batch(scalar_lists, point_lists, POINTS_RISTRETTO, False, engine)

    @staticmethod
    def vartime_multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        return _expect_all(_msm_batch(scalar_lists, point_lists, POINTS_RISTRETTO, False, engine))

    @staticmethod
    def multiscalar_mul_batch(scalar_lists, point_lists, engine=None):
        """RistrettoPoint::multiscalar_mul (ristretto.rs:964-977) for many independent MSMs in one call, constant time in
        the scalars.  An undecodable point or a scalar with bit 255 set raises EngineError."""
        return _msm_batch(scalar_lists, point_lists, POINTS_RISTRETTO, True, engine)

    @staticmethod
    def double_base_batch(a, b, G, H, engine=None):
        eng = engine or default_engine()
        n = len(a) // 32
        rc, out = eng.ristretto_double_base_batch(a, b, G, H, n)
        if rc == 1:
            raise ValueError("G or H is not a valid Ristretto encoding")
        return out

    @staticmethod
    def mul_batch(scalars, points, engine=None):
        """RistrettoPoint * Scalar (ristretto.rs:917-926) for each pair of a 32-byte scalar (bit 255 clear) and a 32-byte
        CompressedRistretto; a single scalar or a single point is used for every item.  Returns the CompressedRistretto
        of the product, or the list.  An undecodable point raises ValueError."""
        return _mul_batch(scalars, points, POINTS_RISTRETTO, False, engine)

    @staticmethod
    def mul_base_batch(scalars, engine=None):
        """RistrettoPoint::mul_base (ristretto.rs:939) for each 32-byte scalar (bit 255 clear), constant time at every batch
        size.  Returns the CompressedRistretto, or the list."""
        return _mul_base_batch(scalars, POINTS_RISTRETTO, False, engine)

    @staticmethod
    def vartime_double_scalar_mul_basepoint_batch(a_list, points, b_list, engine=None):
        """RistrettoPoint::vartime_double_scalar_mul_basepoint (ristretto.rs:1051-1063) for each item: a_i * A_i + b_i * B
        with 32-byte scalars (bit 255 clear) and CompressedRistretto points A_i.  Returns the list of 32-byte
        CompressedRistretto results.  An undecodable point raises ValueError.  Variable time."""
        return _double_base_batch(a_list, points, b_list, POINTS_RISTRETTO, engine)

    @staticmethod
    def from_uniform_bytes_batch(data, engine=None):
        """RistrettoPoint::from_uniform_bytes (ristretto.rs:774-790) for each 64-byte string: the list of 32-byte
        CompressedRistretto encodings."""
        items = [bytes(x) for x in data]
        if any(len(x) != 64 for x in items):
            raise ValueError("from_uniform_bytes takes 64 bytes per item")
        eng = engine or default_engine()
        raw = eng.ristretto_from_uniform_bytes_batch(b"".join(items), len(items))
        return [raw[32 * i:32 * i + 32] for i in range(len(items))]

    @staticmethod
    def hash_from_bytes_batch(messages, engine=None):
        """RistrettoPoint::hash_from_bytes::<Sha512> (ristretto.rs:736-761) for each message: the list of 32-byte
        CompressedRistretto encodings."""
        eng = engine or default_engine()
        flat, offs, n = _flat_messages(messages)
        raw = eng.ristretto_hash_from_bytes_batch(flat, offs, n)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    @staticmethod
    def map_to_curve_batch(data, engine=None):
        """RistrettoPoint::map_to_curve (ristretto/elligator.rs:62-67) for each 32-byte string (bit 255 ignored): the list of
        32-byte CompressedRistretto encodings."""
        _, items = _items(list(data), 32, "map_to_curve inputs")
        if not items:
            return []
        eng = engine or default_engine()
        raw = eng.ristretto_map_to_curve_batch(b"".join(items), len(items))
        return [raw[32 * i:32 * i + 32] for i in range(len(items))]

    @staticmethod
    def lizard_encode_batch(data, engine=None):
        """RistrettoPoint::lizard_encode::<Sha256> (lizard/lizard_ristretto.rs:25-39) for each 16-byte string: the list of
        32-byte CompressedRistretto encodings."""
        _, items = _items(list(data), 16, "Lizard payloads")
        if not items:
            return []
        eng = engine or default_engine()
        raw = eng.ristretto_lizard_encode_batch(b"".join(items), len(items))
        return [raw[32 * i:32 * i + 32] for i in range(len(items))]

    @staticmethod
    def lizard_decode_batch(points, engine=None):
        """RistrettoPoint::lizard_decode::<Sha256> (:43-71) for each 32-byte CompressedRistretto: the 16-byte payload, or
        None when the point is not a Lizard encoding.  An encoding that does not decode raises ValueError."""
        _, items = _items(list(points), 32, "points")
        if not items:
            return []
        eng = engine or default_engine()
        _, raw, st = eng.ristretto_lizard_decode_batch(b"".join(items), len(items))
        if any(s == 2 for s in st):
            raise ValueError("a point does not decode")
        return [raw[16 * i:16 * i + 16] if st[i] == 0 else None for i in range(len(items))]

    @staticmethod
    def map_to_curve_inverse_batch(points, engine=None):
        """RistrettoPoint::map_to_curve_inverse (:213-219) for each 32-byte CompressedRistretto: a list of 16 entries, each the
        32 bytes that map_to_curve takes to the point, or None, in the reference's order.  The candidates depend on the
        representative; a decoded encoding is the one with Z = 1.  An encoding that does not decode raises ValueError."""
        _, items = _items(list(points), 32, "points")
        if not items:
            return []
        eng = engine or default_engine()
        rc, raw, masks = eng.ristretto_map_to_curve_inverse_batch(b"".join(items), len(items))
        if rc == 1:
            raise ValueError("a point does not decode")
        return [[raw[512 * i + 32 * j:512 * i + 32 * j + 32] if masks[i] >> j & 1 else None for j in range(16)]
                for i in range(len(items))]


def verify_batch(messages, signatures, verifying_keys, engine=None):
    """ed25519_dalek::verify_batch (batch.rs:146-251): returns None on Ok, raises SignatureError otherwise."""
    messages, signatures, verifying_keys = list(messages), list(signatures), list(verifying_keys)
    if not (len(messages) == len(signatures) == len(verifying_keys)):
        raise SignatureError(2)                      # batch.rs:152-165 ArrayLength
    eng = engine or default_engine()
    rc = eng.verify_batch_raw(messages, b"".join(signatures), b"".join(verifying_keys))
    if rc != 0:
        raise SignatureError(rc)
    return None
