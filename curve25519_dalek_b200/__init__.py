"""curve25519_dalek_b200 -- host-side mirror of the reference's multiscalar / batch-verify API over
the C ABI of libdalek_b200.so (include/dalek_b200.h).

The product path is the CUDA library; there is no CPU fallback.  Importing this package never
touches the CPU checker used by the tests.  Names follow the reference:
  EdwardsPoint.vartime_multiscalar_mul / optional_multiscalar_mul / multiscalar_mul
      (curve25519-dalek/src/traits.rs:78-262, src/edwards.rs:966-1031)
  RistrettoPoint.multiscalar_mul / vartime_multiscalar_mul (src/ristretto.rs:964-994)
  VartimeEdwardsPrecomputation / VartimeRistrettoPrecomputation (traits.rs:290-406, edwards.rs:1038-1076)
  verify_batch (ed25519-dalek/src/batch.rs:146-251) and its SignatureError values.
  x25519 / x25519_public_keys / X25519_BASEPOINT_BYTES (x25519-dalek/src/x25519.rs:105-110, :385-392)
  EdwardsPoint.to_montgomery_batch (src/edwards.rs:592-612)
  RistrettoPoint.from_uniform_bytes_batch / hash_from_bytes_batch (src/ristretto.rs:736-790)
  EdwardsPoint.hash_to_curve_batch / encode_to_curve_batch (src/edwards.rs:710-750, RFC 9380)
  ed25519_verifying_keys / ed25519_sign / ed25519_sign_prehashed / ed25519_verify_prehashed
      (ed25519-dalek/src/signing.rs:106-171, :312, :566-571; src/verifying.rs:230-257, :424-459)
  EdwardsPoint.mul_batch / mul_clamped_batch / is_small_order_batch / is_torsion_free_batch and RistrettoPoint.mul_batch
      (src/edwards.rs:890-941, :1405-1437; src/ristretto.rs:917-926): constant-time s * P per item, one scalar or one
      point broadcast to the whole batch
  EdwardsPoint / RistrettoPoint .optional_multiscalar_mul_batch / vartime_multiscalar_mul_batch / multiscalar_mul_batch
      (traits.rs:78-262 once per item): many independent MSMs, each with its own scalars and points, in one call
  RistrettoPoint.map_to_curve_batch / lizard_encode_batch / lizard_decode_batch / map_to_curve_inverse_batch
      (src/ristretto/elligator.rs:62-67, src/lizard/lizard_ristretto.rs:25-71, :213-219): Lizard over SHA-256
  EdwardsPoint / RistrettoPoint .vartime_double_scalar_mul_basepoint_batch (src/edwards.rs:1078-1087,
      src/ristretto.rs:1051-1063): a_i A_i + b_i B per item, variable time
  MontgomeryPoint.mul_batch / mul_bits_be_batch / to_edwards_batch / mul_base_batch / mul_clamped_batch /
      mul_base_clamped_batch (src/montgomery.rs:143-268, :484-505): Scalar * MontgomeryPoint, the ladder over any bit
      string of up to 512 bits, Montgomery -> Edwards, and fixed-base u(s B)
  EdwardsPoint.mul_base_batch / mul_base_clamped_batch and RistrettoPoint.mul_base_batch (src/edwards.rs:918-957,
      src/ristretto.rs:939): constant-time s B at every batch size
  ed25519_to_montgomery (ed25519-dalek/src/verifying.rs:476): VerifyingKey::to_montgomery
  EdwardsPoint / RistrettoPoint .add_batch / sub_batch / neg_batch / double_batch / eq_batch / is_identity_batch / sum /
      sum_batch and EdwardsPoint.mul_by_cofactor_batch (src/edwards.rs:501-520, :786-876, :1365-1367; src/ristretto.rs:
      809-908): the group operators, one thread per item, and many segmented sums in one call
  Scalar.from_bytes_mod_order_batch / from_bytes_mod_order_wide_batch / from_canonical_bytes_batch / hash_from_bytes_batch
      / add_batch / sub_batch / mul_batch / neg_batch / div_by_2_batch / invert_each / invert_batch_alloc / sum / sum_batch
      / product / product_batch (src/scalar.rs:235-263, :317-374, :454-476, :617-670, :739-870): arithmetic mod l on
      canonical scalars, one thread per item, and many segmented sums and products in one call
  EdwardsBasepointTable / RistrettoBasepointTable .create / basepoint / mul_base_batch / mul_base_clamped_batch
      (traits.rs:50-74, src/edwards.rs:1127-1243, src/ristretto.rs:1080-1115): resident tables of k points, constant-time
      s * P_{t_i} per item
  VerifyingKeySet .verify_each / verify_prehashed_each / is_weak (ed25519-dalek/src/verifying.rs:167-257, :359-459): k
      VerifyingKeys decompressed and tabulated once on the GPU, each signature verified under its key index
  SigningKeySet .from_seeds / from_keypair_bytes / from_expanded / sign / sign_prehashed / verifying_keys
      (ed25519-dalek/src/signing.rs:106, :140-150, :566-571, :312; hazmat.rs:84-99): k signing keys derived once on the
      GPU, each message signed under its key index
  ed25519_expanded_verifying_keys / ed25519_raw_sign / ed25519_raw_sign_prehashed (ed25519-dalek/src/hazmat.rs:84-99,
      :137, :182; verifying.rs:97-102): signing from ExpandedSecretKey bytes
"""
from .engine import (Engine, MultiEngine, EngineError, EdwardsPoint, RistrettoPoint, MontgomeryPoint, Scalar, SignatureError, verify_batch, default_engine,
                     library_path, load_library, POINTS_COMPRESSED, POINTS_EXTENDED, POINTS_RISTRETTO, POINTS_MONTGOMERY,
                     VartimeEdwardsPrecomputation, VartimeRistrettoPrecomputation, x25519, x25519_public_keys,
                     X25519_BASEPOINT_BYTES, ed25519_verifying_keys, ed25519_sign, ed25519_sign_prehashed,
                     ed25519_verify_prehashed, ed25519_to_montgomery, EdwardsBasepointTable, RistrettoBasepointTable,
                     VerifyingKeySet, SigningKeySet, ed25519_expanded_verifying_keys, ed25519_raw_sign,
                     ed25519_raw_sign_prehashed)

__all__ = ["Engine", "MultiEngine", "EngineError", "EdwardsPoint", "RistrettoPoint", "MontgomeryPoint", "Scalar", "SignatureError", "verify_batch", "default_engine",
           "library_path", "load_library", "POINTS_COMPRESSED", "POINTS_EXTENDED", "POINTS_RISTRETTO", "POINTS_MONTGOMERY",
           "VartimeEdwardsPrecomputation", "VartimeRistrettoPrecomputation", "x25519", "x25519_public_keys",
           "X25519_BASEPOINT_BYTES", "ed25519_verifying_keys", "ed25519_sign", "ed25519_sign_prehashed",
           "ed25519_verify_prehashed", "ed25519_to_montgomery", "EdwardsBasepointTable", "RistrettoBasepointTable",
           "VerifyingKeySet", "SigningKeySet", "ed25519_expanded_verifying_keys", "ed25519_raw_sign",
           "ed25519_raw_sign_prehashed"]
