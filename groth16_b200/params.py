"""Field moduli and limb counts of the supported curves: the pairing curves BLS12-381, BN254 and BLS12-377 (SURVEY.md
section 2b) and BW6-761, the outer curve of BLS12-377 recursion.

Only what the host-side codecs need; the CUDA side has its own generated table (csrc/g16_constants.h)."""
from dataclasses import dataclass


@dataclass(frozen=True)
class CurveParams:
    name: str
    cid: int            # curve id at the C ABI (include/g16b200.h)
    r: int              # scalar field modulus
    q: int              # base field modulus
    fr_generator: int   # Fr::GENERATOR (coset offset, r1cs_to_qap.rs:204)
    two_adicity: int
    g2_over_fq: bool = False   # G2 coordinates in Fq itself (BW6-761) instead of Fq2

    @property
    def fq_limbs(self) -> int:
        return (self.q.bit_length() + 63) // 64

    @property
    def fr_limbs(self) -> int:
        return (self.r.bit_length() + 63) // 64

    @property
    def g2_limbs(self) -> int:
        """u64 limbs of one G2 affine point"""
        return (2 if self.g2_over_fq else 4) * self.fq_limbs


BLS12_381 = CurveParams(
    "bls12_381", 0,
    0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
    0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
    7, 32)
BN254 = CurveParams(
    "bn254", 1,
    21888242871839275222246405745257275088548364400416034343698204186575808495617,
    21888242871839275222246405745257275088696311157297823662689037894645226208583,
    5, 28)
BLS12_377 = CurveParams(
    "bls12_377", 2,
    8444461749428370424248824938781546531375899335154063827935233455917409239041,
    258664426012969094010652733694893533536393512754914660539884262666720468348340822774968888139573360124440321458177,
    22, 47)

# BW6-761: r is BLS12-377's q.  G1: y^2 = x^3 - 1, G2: y^2 = x^3 + 4, both over Fq.
BW6_761 = CurveParams(
    "bw6_761", 3,
    BLS12_377.q,
    0x122e824fb83ce0ad187c94004faff3eb926186a81d14688528275ef8087be41707ba638e584e91903cebaff25b423048689c8ed12f9fd9071dcd3dc73ebff2e98a116c25667a8f8160cf8aeeaf0a437e6913e6870000082f49d00000000008b,
    15, 46, g2_over_fq=True)

CURVES = {c.name: c for c in (BLS12_381, BN254, BLS12_377, BW6_761)}


def get_curve(curve) -> CurveParams:
    if isinstance(curve, CurveParams):
        return curve
    if isinstance(curve, str):
        return CURVES[curve]
    if hasattr(curve, "name"):
        return CURVES[curve.name]
    raise KeyError(curve)


# Fixed points of prime order r in G1 / G2, used as the "random group generators" of the trusted setup
# (generator.rs:26-32 samples them; any r-torsion points are valid).  Derived once by hashing to an x coordinate and
# clearing the cofactor; tests/test_constants.py re-derives them with the oracle and checks order and curve equation.
GENERATORS = {
    "bls12_381": dict(
        g1=(0x7225faa9ea1508c4c911e95beee000273bcbcbbd1d41ce0f18e8659251c0df081f9327b47e7a275f5a8031e433aa871,
            0x1949d82fc886648068a620dbb0a53b4c66213f267efa964cc41d733acdea86ce2c00e22e3202c3c594f339f30c2e3051),
        g2=((0x14e99e3b657acbd60979fa3525ae77af164a311785d46a08e67c54463326a88c60f04d6ded6397b2731df815d95892ca,
             0xa4601a9a48444765251e2a65f0b5619c3ea7290b0d3f6da7a8f3363808b58bb9e978796daba529742b6458d9e939b23),
            (0x1254a4d6508c091d0c5099f847013293e8d60d995850c5e88b1f18a7ef33f05d80bd1fedd8b272c6d123bdbfc18cb40d,
             0x4f838240ae2b657dcbd587add1ee8bde44e8802453d401454eec303e0e0bdfdf2fc11f9c642b8e2857205c8e32f01be))),
    "bn254": dict(
        g1=(0x2fda4996c18c5417c7ea845438e13c5d8c7e190a961ff9abbf8263e27d10ae7c,
            0x11911b5eaf5b93b8f1c774ba78cf95255929d38f32bfaad3167451e7c220715d),
        g2=((0x1df968558dbed90f366d524d5060557cc2f5b61c513ff08d463bc2843848b870,
             0x15ea7aac5c64a54af33865da65cf9ae6bbd4a0dd0b08317fc4aca44cd4560c50),
            (0xff98893b3d0be07b26b9485d5237dfcb32473d07a50d810132babe65d792aeb,
             0x2ea59f614a18e9f222cde53f20176036f654442bbd915ee616b7c422c0f8d69f))),
    "bls12_377": dict(
        g1=(0xe09f3eb12c7f3e7b77a61139ee7e62bb97ff9d88b8df1791fcf66b0dec04e4f24be4e0989fae248218a13843ed03d9,
            0x18144cece60d3a8fb0b6d28d6f8fe3a915e2be042f16b230110fb6b4a133d233236e7a189192b3dc4e31109664765d1),
        g2=((0x12cd874591f305b74d3cda047a5f555e752911ced088131536de5023ee8c1aed7aadb3ff7c15f6357f832f9698b963d,
             0x895a8006e7536bdf93f71f27bd5b280fa531cc66f63449312a91ec01c684a6ccff1ebd00e2931c19b0ac9bf61d4f68),
            (0x17663bd2b96d697799583fe676e7df81723dc2c223265cc2685c69e2b7d4c8464c342be5846f0eeeeec44de888db212,
             0x1b49e02eade86f46ff617db109925f68fc7bd69f1dbcbae76ff26e3388801324d585e56fbfb1cc438029a7a8b7f6b3))),
    # G2 over Fq: g2 is an (x, y) pair like g1.  A recipe of its own, not the other curves' (a 256-bit hash, too short for a
    # 761-bit x): x = the 1024-bit little-endian integer of sha512("bw6_761-g<k>:<i>") repeated twice, mod q, for the first i
    # with a curve point (the smaller root y), times the 384-bit cofactor.  tests/test_bw6_cpu.py re-derives both.
    "bw6_761": dict(
        g1=(0xc4b9f2bdb719ce82628aeb2dce695848ccd7d8ada4eb2389732d498070cb23548fe3477cefa0b8a1189abe80b7350cec7944f4b1b70efd816a33f2f9cc136b6b7ff59253118d154eb7284e3321d6176fe081075ab3d349f5a74d54640a1b2f,
            0x29430bee0dc548df82627abd2d312248f1bff387ad5c5f8197e50ae8e9d701b5f5ef655b751e9abaa61a3ada0864feb5e19972a3a1e38e501291719e1925ddcb209d8fdde82fc687daeefa1de84d80ded2f1bc29eb85547911897400f7dc23),
        g2=(0x85ba4ee833fa16b37d0b1a861dc4caaa5b65ea073d65de92306440aa11225b1c66feb22afe5b2f76184642dd572e76be86b8f6e0a57af8864529d02b1cb6734209c828d3ff359daa153866695a707036dc8f13774c3178888713705752b8f1,
            0xa5d36491ece4b262680ab6a294cc5b716290462eba70d0f42a2443599fa80df90c35fe3479e5e3159cfb60719ac1634eb415b9e088c315f506e6aec397a12a6c142c2fcb39d70fc2615d32ac1a2fae190dfaba433796f107f82b9cf2964035)),
}
