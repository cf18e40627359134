#!/usr/bin/env python3
"""Write tests/golden/hash_to_curve.json: the reference's known answers for hashing into the group, copied as data, and
edge vectors computed by the independent model (tests/h2c_model.py), each labelled with what it exercises.

The generator asserts that the model reproduces every reference known answer and that the C oracle
(tests/host/h2c_oracle.c) agrees with every vector.  Known answers (curve25519-dalek):
  elligator_vs_ristretto_sage and one_way_map (src/ristretto/elligator.rs:76-388);
  RFC_HASH_TO_CURVE_KAT / RFC_ENCODE_TO_CURVE_KAT (src/edwards.rs, RFC 9380 J.5.1 / J.5.2);
  RFC_HASH_TO_FIELD_KAT, RFC_HASH_TO_FIELD_KAT_2 and FROM_BYTES_WIDE_KAT_BIG (src/field.rs)."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import h2c_model as M  # noqa: E402

p = M.p
DST_RO = b"QUUX-V01-CS02-with-edwards25519_XMD:SHA-512_ELL2_RO_"
DST_NU = b"QUUX-V01-CS02-with-edwards25519_XMD:SHA-512_ELL2_NU_"
RFC_MSGS = [b"", b"abc", b"abcdef0123456789", b"q128_" + b"q" * 128, b"a512_" + b"a" * 512]

SAGE = [  # (r0, CompressedRistretto) of elligator_vs_ristretto_sage
    ("b8f98731fd7b597143a006ef0769d329c0f9b939096646c60f7f071aa0668647", "b09ded61421d8ca6a85e1a9dd4d8e5a0c3f6e8efa9703fc1402098450bbef656"),
    ("e50ef1e34b09763c8099e215b7d95b886200e79c7c4d528b8e86a4a9a93efa34", "ea8d4dcbb5e1fa4aab3e0f764ed49613830ebceec2f48d8aa6a2537ae4c9131a"),
    ("736d24dcb4df6306cca9131da944541715 6dbd957fcd5b66ac2370238645ba22".replace(" ", ""), "e8e7335c05a85024adb36844ba9544288caa1b67638c15f22b3efa86d0ff3d59"),
    ("1031606babc7a4098110403ef13f84add1a070d769329d51fd69019ae5197853", "d0788c81b1b3ed9ffca01c0dce05d3f1c0da016182f114a9772ef61d4f504d54"),
    ("9c83a1a2ecfb05bba7ab11b294d25acf56154fa1a7d7ea0188f2b6f826554f56", "ca0bec913a0cb59dd106d5584b930b77bf8b2f8e212499c1dfb7b208cd78f86e"),
    ("fbb17c3612654bebf5ba132e859de5400a88b5b94e90fea789316b0a3d0a1519", "1a42e743cbaf748220883efdd72e05d6a6f86cedd847f4ad488552068ff06829"),
    ("e8c11444f04dba4db7282c56961fc6d44c5103d9c5087e807e98a4d0992cbd4d", "289d6660c9dfc8c596b56a53677e8f2191e64e06ab92d28f7005f517b78a1278"),
    ("ade595b125e61e453d38acbedb73a7c247863b4b1cf4761aa26140100fbd1e40", "dc251bcbefc4b0832542bcf3b9fa7117a7d39af3a8d736ab9f24c3510d962b2b"),
    ("6a473d6bfa752a975bcad46434bcbe157dda1f12fdf1a08539f203a4bd446f4b", "e879b0deb7c49f5aeec1693465a7f4aa7972c40643985 0b9dd075369b0d0e079".replace(" ", "")),
    ("70ccb65adcc67849ad6bc111e328a224968deb37acb70c27c2882b99f4765b59", "e2b5b734f1a33db3ddcfdc49f5f219ec4354b3dea73ea7b620095c1ea57fcc44"),
    ("6f18cb7bfebd0ba233c4a388cc8f0ade217051cd2223 08425a06a43aaab12219".replace(" ", ""), "e27710f2c88bf0570bde5c929cf32e77413b01f85cb732af5728ce35d0dc940d"),
    ("e1b71e34ec5206b76d19e3b5195229c1504da150f2cb4fcc88f5836eed6a033a", "46f04f70369de4924a7ad858e83e9e0d0e927375b0de5ae1f4175ebe96078860"),
    ("cff626381e56b05a1bc83d2add1b38d24fb2bd7844c178a74db935c57c80bf7e", "1647f1672dc1c390b7659a322744316e332c3e00e5714851a81d496a66288418"),
    ("0188d750f02e3f9310f4e6cf52bd4a326aa98a561e83d6caa67dfbe462182415", "c4856b0b82694a21ccab85ddaec1f12426b3c46bdbb9b5fde42f9b2ae749294e"),
    ("d2cfe4389b74cf3654c3fbd7f9c7744b6defc4fbc2f6fce446929c231927f104", "3affe1c573d0a08f27c552458feb5caa4a28390babe31ab9d9cf5ab9c5be233c"),
    ("22747b0908285dbd0967396742e303029d6b86dbca4ae69a4e6bdbc3d60e5450", "582b5c76df886991eeba7308d67099fd266ccde69d820b426555fd6e6e0e9470"),
]
ONE_WAY = [  # (64-byte input, CompressedRistretto) of one_way_map
    ("5d1be09e3d0c82fc538112490e35701979d99e06ca3e2b5b54bffe8b4dc772c14d98b696a1bbfb5ca32c436cc61c16563790306c79eaca7705668b47dffe5bb6",
     "3066f82a1a747d45120d1740f14358531a8f04bbffe6a819f86dfe50f44a0a46"),
    ("f116b34b8f17ceb56e8732a60d913dd10cce47a6d53bee9204be8b44f6678b270102a56902e2488c46120e9276cfe54638286b9e4b3cdb470b542d46c2068d38",
     "f26e5b6f7d362d2d2a94c5d0e7602cb4773c95a2e5c31a64f133189fa76ed61b"),
    ("8422e1bbdaab52938b81fd602effb6f89110e1e57208ad12d9ad767e2e25510c27140775f9337088b982d83d7fcf0b2fa1edffe51952cbe7365e95c86eaf325c",
     "006ccd2a9e6867e6a2c5cea83d3302cc9de128dd2a9a57dd8ee7b9d7ffe02826"),
    ("ac22415129b61427bf464e17baee8db65940c233b98afce8d17c57beeb7876c2150d15af1cb1fb824bbd14955f2b57d08d388aab431a391cfc33d5bafb5dbbaf",
     "f8f0c87cf237953c5890aec3998169005dae3eca1fbb04548c635953c817f92a"),
    ("165d697a1ef3d5cf3c38565beefcf88c0f282b8e7dbd28544c483432f1cec7675debea8ebb4e5fe7d6f6e5db15f15587ac4d4d4a1de7191e0c1ca6664abcc413",
     "ae81e7dedf20a497e10c304a765c1767a42d6e06029758d2d7e8ef7cc4c41179"),
    ("a836e6c9a9ca9f1e8d486273ad56a78c70cf18f0ce10abb1c7172ddd605d7fd2979854f47ae1ccf204a33102095b4200e5befc0465accc263175485f0e17ea5c",
     "e2705652ff9f5e44d3e841bf1c251cf7dddb77d140870d1ab2ed64f1a9ce8628"),
    ("2cdc11eaeb95daf01189417cdddbf95952993aa9cb9c640eb5058d09702c74622c9965a697a3b345ec24ee56335b556e677b30e6f90ac77d781064f866a3c982",
     "80bd07262511cdde4863f8a7434cef696750681cb9510eea557088f76d9e5065"),
    # the last four all map to one point (the elligator.rs comments: inputs equal modulo p and bit 255)
    ((b"\xed" + b"\xff" * 31 + b"\x12" + bytes(31)).hex(), "304282791023b73128d277bdcb5c7746ef2eac08dde9f2983379cb8e5ef0517f"),
    ((b"\xed" + b"\xff" * 30 + b"\x7f" + b"\xff" * 32).hex(), "304282791023b73128d277bdcb5c7746ef2eac08dde9f2983379cb8e5ef0517f"),
    ((bytes(31) + b"\x80" + b"\xff" * 31 + b"\x7f").hex(), "304282791023b73128d277bdcb5c7746ef2eac08dde9f2983379cb8e5ef0517f"),
    ((bytes(32) + b"\x12" + bytes(30) + b"\x80").hex(), "304282791023b73128d277bdcb5c7746ef2eac08dde9f2983379cb8e5ef0517f"),
]
H2C_KAT = [  # RFC 9380 J.5.1 (x, y) big-endian hex
    ("3c3da6925a3c3c268448dcabb47ccde5439559d9599646a8260e47b1e4822fc6", "09a6c8561a0b22bef63124c588ce4c62ea83a3c899763af26d795302e115dc21"),
    ("608040b42285cc0d72cbb3985c6b04c935370c7361f4b7fbdb1ae7f8c1a8ecad", "1a8395b88338f22e435bbd301183e7f20a5f9de643f11882fb237f88268a5531"),
    ("6d7fabf47a2dc03fe7d47f7dddd21082c5fb8f86743cd020f3fb147d57161472", "53060a3d140e7fbcda641ed3cf42c88a75411e648a1add71217f70ea8ec561a6"),
    ("5fb0b92acedd16f3bcb0ef83f5c7b7a9466b5f1e0d8d217421878ea3686f8524", "2eca15e355fcfa39d2982f67ddb0eea138e2994f5956ed37b7f72eea5e89d2f7"),
    ("0efcfde5898a839b00997fbe40d2ebe950bc81181afbd5cd6b9618aa336c1e8c", "6dc2fc04f266c5c27f236a80b14f92ccd051ef1ff027f26a07f8c0f327d8f995"),
]
E2C_KAT = [  # RFC 9380 J.5.2
    ("1ff2b70ecf862799e11b7ae744e3489aa058ce805dd323a936375a84695e76da", "222e314d04a4d5725e9f2aff9fb2a6b69ef375a1214eb19021ceab2d687f0f9b"),
    ("5f13cc69c891d86927eb37bd4afc6672360007c63f68a33ab423a3aa040fd2a8", "67732d50f9a26f73111dd1ed5dba225614e538599db58ba30aaea1f5c827fa42"),
    ("1dd2fefce934ecfd7aae6ec998de088d7dd03316aa1847198aecf699ba6613f1", "2f8a6c24dd1adde73909cada6a4a137577b0f179d336685c4a955a0a8e1a86fb"),
    ("35fbdc5143e8a97afd3096f2b843e07df72e15bfca2eaf6879bf97c5d3362f73", "2af6ff6ef5ebba128b0774f4296cb4c2279a074658b083b8dcca91f57a603450"),
    ("6e5e1f37e99345887fc12111575fc1c3e36df4b289b8759d23af14d774b66bff", "2c90c3d39eb18ff291d33441b35f3262cdd307162cc97c31bfcc7a4245891a37"),
]
H2F_KAT = [  # RFC_HASH_TO_FIELD_KAT (NU DST, count 1), big-endian
    "7f3e7fb9428103ad7f52db32f9df32505d7b427d894c5093f7a0f0374a30641d",
    "09cfa30ad79bd59456594a0f5d3a76f6b71c6787b04de98be5cd201a556e253b",
    "475ccff99225ef90d78cc9338e9f6a6bb7b17607c0c4428937de75d33edba941",
    "049a1c8bd51bcb2aec339f387d1ff51428b88d0763a91bcdf6929814ac95d03d",
    "3cb0178a8137cefa5b79a3a57c858d7eeeaa787b2781be4a362a2f0750d24fa0",
]
H2F_KAT_2 = [  # RFC_HASH_TO_FIELD_KAT_2 (RO DST, count 2)
    ("03fef4813c8cb5f98c6eef88fae174e6e7d5380de2b007799ac7ee712d203f3a", "780bdddd137290c8f589dc687795aafae35f6b674668d92bf92ae793e6a60c75"),
    ("5081955c4141e4e7d02ec0e36becffaa1934df4d7a270f70679c78f9bd57c227", "005bdc17a9b378b6272573a31b04361f21c371b256252ae5463119aa0b925b76"),
    ("285ebaa3be701b79871bcb6e225ecc9b0b32dff2d60424b4c50642636a78d5b3", "2e253e6a0ef658fedb8e4bd6a62d1544fd6547922acb3598ec6b369760b81b31"),
    ("4fedd25431c41f2a606952e2945ef5e3ac905a42cf64b8b4d4a83c533bf321af", "02f20716a5801b843987097a8276b6d869295b2e11253751ca72c109d37485a9"),
    ("6e34e04a5106e9bd59f64aba49601bf09d23b27f7b594e56d5de06df4a4ea33b", "1c1c2cb59fc053f44b86c5d5eb8c1954b64976d0302d3729ff66e84068f5fd96"),
]
WIDE_KAT = [  # FROM_BYTES_WIDE_KAT_BIG: (64 bytes, canonical encoding)
    ("77b663085cac0e916f40dbeea5116f201816406e68ccf01b32a97162ae1d5bf95d0d01c2c72fbeeb27a635b85b715d5ce6f74118a60a7aec53c798ad648a482f",
     "62b38bd402c4498f5cead14643e54dd649e20a0810610e36a73f1f27a0a81f7e"),
    ("d437c75ec79886650243a79c62933bb307eb12ff16d05db4a6a8a877f4a91abb6eeb64d2e20519c0217993a1dc5639283a06639985a2c892208171503335afb5",
     "3d2ec29972783de9043e8b982278beaba9d7c5c3ebef257e7cd38168928f1c33"),
    ("6daa9e1abe6c604fb6e841c04bf90a6ef88aef6b1eab17dd44f7207ef472cd2d54bac849f703e64f36e5677e7e86b82be7d26aa220daf1f208bb36dcc1a12338",
     "28546a0e7303852bc6eead8312f06eeb48d9ca87f60bfeec98ba402ebb751703"),
    ("c3920e326dbf806a50105be78263c1dc9390fb4741587b250cd758c2bfa3ed70faedbbc5f9b1d024e00fe7d7daf796866853f42e72d638e6533c5eb5b7caf3c6",
     "40eaf38b802a7be1956ba7f3fe2d2ad717f23f40342deb5180cb55ae04bb1d79"),
    ("23f143c72ead6c0f336b4e746a06921f0eb180002e8ce916d196de16216788617c6aeb90a074a85196f0381375011248927c1215e9ec65b382a6ec556fb3f504",
     "b1bf354a04fd6d2e8321c24ecb3d3ed2c42e3f21c7b60ab8374effd7a709011e"),
]


def xy_to_compressed(xh, yh):
    x, y = int(xh, 16), int(yh, 16)
    return (y | ((x & 1) << 255)).to_bytes(32, "little").hex()


def b32(x):
    return x.to_bytes(32, "little")


def generate():
    g = {"note": "written by tests/golden/make_hash_to_curve_golden.py; reference known answers copied as data, the rest "
                 "computed by tests/h2c_model.py", "dst_ro": DST_RO.hex(), "dst_nu": DST_NU.hex()}
    # ---- reference known answers, reproduced by the model
    g["ristretto_elligator_sage"] = [{"r0": r, "out": o} for r, o in SAGE]
    for v in g["ristretto_elligator_sage"]:
        assert M.ristretto_elligator(bytes.fromhex(v["r0"])).hex() == v["out"]
    g["one_way_map"] = [{"in": i, "out": o} for i, o in ONE_WAY]
    for v in g["one_way_map"]:
        assert M.from_uniform_bytes(bytes.fromhex(v["in"])).hex() == v["out"]
    g["rfc9380_hash_to_curve"] = [{"msg": m.hex(), "out": xy_to_compressed(x, y)} for m, (x, y) in zip(RFC_MSGS, H2C_KAT)]
    g["rfc9380_encode_to_curve"] = [{"msg": m.hex(), "out": xy_to_compressed(x, y)} for m, (x, y) in zip(RFC_MSGS, E2C_KAT)]
    for v in g["rfc9380_hash_to_curve"]:
        assert M.hash_to_curve(bytes.fromhex(v["msg"]), DST_RO).hex() == v["out"]
    for v in g["rfc9380_encode_to_curve"]:
        assert M.encode_to_curve(bytes.fromhex(v["msg"]), DST_NU).hex() == v["out"]
    g["rfc9380_hash_to_field_1"] = [{"msg": m.hex(), "u": [b32(int(h, 16)).hex()]} for m, h in zip(RFC_MSGS, H2F_KAT)]
    g["rfc9380_hash_to_field_2"] = [{"msg": m.hex(), "u": [b32(int(a, 16)).hex(), b32(int(b, 16)).hex()]}
                                    for m, (a, b) in zip(RFC_MSGS, H2F_KAT_2)]
    for v in g["rfc9380_hash_to_field_1"]:
        assert [b32(x).hex() for x in M.hash_to_field(bytes.fromhex(v["msg"]), DST_NU, 1)] == v["u"]
    for v in g["rfc9380_hash_to_field_2"]:
        assert [b32(x).hex() for x in M.hash_to_field(bytes.fromhex(v["msg"]), DST_RO, 2)] == v["u"]
    g["from_bytes_wide"] = [{"in": i, "out": o} for i, o in WIDE_KAT]
    for v in g["from_bytes_wide"]:
        assert b32(M.from_bytes_wide(bytes.fromhex(v["in"]))).hex() == v["out"]

    # ---- model edge vectors
    rnd = random.Random(20261015)
    halves = {"0": 0, "1": 1, "p-1": p - 1, "p": p, "p+1": p + 1, "2^255-1": 2**255 - 1}
    edge = []
    for n1, h1 in halves.items():
        for n2, h2 in halves.items():
            for top in (0, 1):
                raw = b32(h1 | (top << 255)) + b32(h2 | (top << 255))
                edge.append({"label": "halves %s | %s, bit 255 %s" % (n1, n2, "set" if top else "clear"), "in": raw.hex()})
    dz = M.d_zero_halves()
    labels = ["D = 0: r = -d, +root", "D = 0: r = -d, -root", "D = 0: r = -1/d, +root", "D = 0: r = -1/d, -root"]
    g["d_zero_halves"] = [b32(x).hex() for x in dz]
    for lab, x in zip(labels, dz):
        other = rnd.randrange(p)
        edge.append({"label": lab + " (first half)", "in": (b32(x) + b32(other)).hex()})
        edge.append({"label": lab + " (second half)", "in": (b32(other) + b32(x)).hex()})
        edge.append({"label": lab + " (both halves)", "in": (b32(x) + b32(x)).hex()})
    # Ns_D_is_sq survey over random halves
    survey = {"square": 0, "nonsquare": 0}
    sq_halves, nsq_halves = [], []
    for _ in range(1024):
        r0 = rnd.randrange(2**255)
        if M.ns_d_is_square(r0 % p):
            survey["square"] += 1
            sq_halves.append(r0)
        else:
            survey["nonsquare"] += 1
            nsq_halves.append(r0)
    g["ns_d_is_sq_survey"] = dict(survey, total=1024)
    for a, b in zip(sq_halves[:8], nsq_halves[:8]):
        edge.append({"label": "Ns_D_is_sq true | false", "in": (b32(a) + b32(b)).hex()})
        edge.append({"label": "Ns_D_is_sq false | true", "in": (b32(b) + b32(a)).hex()})
    edge.append({"label": "Ns_D_is_sq true | true", "in": (b32(sq_halves[8]) + b32(sq_halves[9])).hex()})
    edge.append({"label": "Ns_D_is_sq false | false", "in": (b32(nsq_halves[8]) + b32(nsq_halves[9])).hex()})
    for v in edge:
        v["out"] = M.from_uniform_bytes(bytes.fromhex(v["in"])).hex()
    g["from_uniform_edges"] = edge

    hfb = []
    for n in (0, 1, 111, 112, 127, 128, 129, 239, 240, 1000):
        m = bytes(rnd.randrange(256) for _ in range(n))
        hfb.append({"label": "message of %d bytes" % n, "msg": m.hex(), "out": M.hash_from_bytes(m).hex()})
    g["hash_from_bytes_lengths"] = hfb

    # XMD block boundaries: msg_prime = 128 + len + 3 + dst_len + 1 bytes; b_1 input = 64 + 1 + dst_len + 1 bytes
    xmd = []
    for dlen in (1, 45, 46, 124, 125, 255):
        dst = bytes(rnd.randrange(256) for _ in range(dlen))
        tail = 4 + dlen                                  # msg_prime bytes after the message, Z_pad excluded
        lens = sorted({0, 1, 32} | {max(0, k * 128 - tail + e) for k in (1, 2) for e in (-17, -16, -1, 0, 1)})
        for mlen in lens:
            m = bytes(rnd.randrange(256) for _ in range(mlen))
            xmd.append({"label": "dst_len %d, message of %d bytes (msg_prime %d bytes)" % (dlen, mlen, 128 + mlen + tail),
                        "msg": m.hex(), "dst": dst.hex(),
                        "uniform_48": M.expand_message_xmd(m, dst, 48).hex(), "uniform_96": M.expand_message_xmd(m, dst, 96).hex(),
                        "hash_to_curve": M.hash_to_curve(m, dst).hex(), "encode_to_curve": M.encode_to_curve(m, dst).hex()})
    g["xmd_boundaries"] = xmd

    # map-level inputs no hash reaches in practice: u = 0 and the other tv1 = xd yd = 0 inputs of the rational map
    maps = [{"label": "u = 0", "u": b32(0).hex()}]
    J = M.J
    for lab, sq in (("x1 = -1", (J - 1) * M.inv(2) % p), ("x2 = -1", M.inv(2 * (J - 1)) % p)):
        ok, r = M.sqrt_ratio_m1(sq, 1)
        if ok:
            for s, u in (("+", r), ("-", (p - r) % p)):
                if M.exceptional(u):
                    maps.append({"label": "%s, u = %sroot" % (lab, s), "u": b32(u).hex()})
    for k in range(4):
        maps.append({"label": "random u", "u": b32(rnd.randrange(p)).hex()})
    for v in maps:
        u = int.from_bytes(bytes.fromhex(v["u"]), "little")
        v["exceptional"] = M.exceptional(u)
        v["out"] = M.map_to_curve_compressed(u).hex()
    g["map_to_curve"] = maps
    return g


def check_oracle(g):
    import h2c_oracle
    o = h2c_oracle.load()
    ro, nu = DST_RO, DST_NU
    for v in g["ristretto_elligator_sage"]:
        assert o.ristretto_elligator(bytes.fromhex(v["r0"])).hex() == v["out"]
    for v in g["one_way_map"] + g["from_uniform_edges"]:
        assert o.from_uniform_bytes(bytes.fromhex(v["in"])).hex() == v["out"], v.get("label")
    for v in g["rfc9380_hash_to_curve"]:
        assert o.hash_to_curve(bytes.fromhex(v["msg"]), ro).hex() == v["out"]
    for v in g["rfc9380_encode_to_curve"]:
        assert o.encode_to_curve(bytes.fromhex(v["msg"]), nu).hex() == v["out"]
    for v in g["rfc9380_hash_to_field_1"]:
        assert [u.hex() for u in o.hash_to_field(bytes.fromhex(v["msg"]), nu, 1)] == v["u"]
    for v in g["rfc9380_hash_to_field_2"]:
        assert [u.hex() for u in o.hash_to_field(bytes.fromhex(v["msg"]), ro, 2)] == v["u"]
    for v in g["from_bytes_wide"]:
        assert o.from_bytes_wide(bytes.fromhex(v["in"])).hex() == v["out"]
    for v in g["hash_from_bytes_lengths"]:
        assert o.hash_from_bytes(bytes.fromhex(v["msg"])).hex() == v["out"]
    for v in g["xmd_boundaries"]:
        m, dst = bytes.fromhex(v["msg"]), bytes.fromhex(v["dst"])
        assert o.expand_message_xmd(m, dst, 48).hex() == v["uniform_48"]
        assert o.expand_message_xmd(m, dst, 96).hex() == v["uniform_96"]
        assert o.hash_to_curve(m, dst).hex() == v["hash_to_curve"]
        assert o.encode_to_curve(m, dst).hex() == v["encode_to_curve"]
    for v in g["map_to_curve"]:
        assert o.map_to_curve(bytes.fromhex(v["u"])).hex() == v["out"], v["label"]


def render(g):
    return json.dumps(g, indent=1, sort_keys=True) + "\n"


if __name__ == "__main__":
    g = generate()
    check_oracle(g)
    path = os.path.join(HERE, "hash_to_curve.json")
    with open(path, "w") as f:
        f.write(render(g))
    print("wrote", path, {k: len(v) for k, v in g.items() if isinstance(v, list)}, g["ns_d_is_sq_survey"])
