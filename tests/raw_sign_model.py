"""A model of ed25519-dalek's hazmat signing from ExpandedSecretKey bytes, built from the C oracle's primitives (SHA-512,
the wide reduction, scalar arithmetic mod l, scalar multiplication and compression).  TEST INFRASTRUCTURE ONLY.

  ExpandedSecretKey::from_bytes (hazmat.rs:84-99): scalar = clamp(bytes[0..32]) mod l, hash_prefix = bytes[32..64]
  VerifyingKey::from(&esk) (verifying.rs:97-102): compress([scalar]B)
  raw_sign (signing.rs:854-904) / raw_sign_prehashed (signing.rs:917-976): r = H([dom2 ||] prefix || M), R = [r]B,
  k = H([dom2 ||] R || vk || M) with vk hashed as given, s = k scalar + r"""


def clamp(lo):
    """clamp_integer (scalar.rs:1407-1412)."""
    a = bytearray(lo)
    a[0] &= 248
    a[31] &= 127
    a[31] |= 64
    return bytes(a)


def dom2(context):
    return b"SigEd25519 no Ed25519 collisions" + bytes([1, len(context)]) + context


class RawSignModel:
    def __init__(self, orc):
        self.orc = orc
        self.B = orc.basepoint()

    def scalar(self, esk):
        return self.orc.sc_op1("scalar_reduce", clamp(esk[:32]))

    def verifying_key(self, esk):
        return self.orc.compress(self.orc.scalarmul(self.scalar(esk), self.B))

    def _sign(self, esk, msg, vk, dom):
        o = self.orc
        r = o.scalar_from_wide(o.sha512(dom + esk[32:] + msg))
        R = o.compress(o.scalarmul(r, self.B))
        k = o.scalar_from_wide(o.sha512(dom + R + vk + msg))
        return R + o.sc_op2("scalar_add", o.sc_op2("scalar_mul", k, self.scalar(esk)), r)

    def raw_sign(self, esk, msg, vk):
        return self._sign(esk, msg, vk, b"")

    def raw_sign_prehashed(self, esk, prehash, vk, context=b""):
        return self._sign(esk, prehash, vk, dom2(context))
