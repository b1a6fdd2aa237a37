"""Per-base consensus qualities (extension: `qualities=True`, `kindel consensus --fastq`; the reference has none).

The device writes the quality of every emitted base (K2q, kindel_b200/csrc/assemble.cu); the host needs the same rule
for the few characters it decides itself -- inserted strings -- and restates it here with the same table:

    D = the depth, k = the support of what is emitted; Q = 0 when k == 0, else the largest q in 0..60 with
    (double)(D - k + 1) * TEN[q] <= (double)(D + 2),   TEN[q] = the correctly rounded double of 10^(q/10)

(D - k + 1) / (D + 2) is the rule of succession's posterior mean of the disagreement rate, so Q grows with agreement
and with depth.  The compare is one correctly rounded multiply, as in CUDA, so host and device agree bit for bit.
Quality characters are Phred+33: chr(33 + Q).

The quality vote (extension: `quality_vote=True`, `kindel consensus --quality-vote`) weights each counted base of
Phred q by WEIGHT[min(q, 93)], a constant table (its formula: DESIGN.md section 1, thirteenth extension): the
log-likelihood ratio, in 1/65536 Phred, of "the true base is the one read" against "it is one particular other base".
K11w sums it per slot and base, and K2w votes with the sums (include/kindel_b200.h kdl_quality_weights /
kdl_vote_quality); the device holds the same table (kQualWeight, kindel_b200/csrc/quality.cu).
"""
from __future__ import annotations

QUAL_MAX = 60

WEIGHT = (
    0, 0, 160037, 311335, 430336, 532174, 623571, 708096,
    787861, 864214, 938059, 1010026, 1080568, 1150020, 1218628, 1286580,
    1354022, 1421062, 1487787, 1554264, 1620546, 1686672, 1752677, 1818584,
    1884415, 1950185, 2015906, 2081590, 2147243, 2212872, 2278481, 2344076,
    2409659, 2475232, 2540797, 2606356, 2671911, 2737461, 2803009, 2868554,
    2934098, 2999640, 3065180, 3130720, 3196259, 3261797, 3327335, 3392873,
    3458410, 3523947, 3589483, 3655020, 3720556, 3786093, 3851629, 3917165,
    3982701, 4048238, 4113774, 4179310, 4244846, 4310382, 4375918, 4441454,
    4506990, 4572526, 4638062, 4703598, 4769134, 4834670, 4900206, 4965742,
    5031278, 5096814, 5162350, 5227886, 5293422, 5358958, 5424494, 5490030,
    5555566, 5621102, 5686638, 5752174, 5817710, 5883246, 5948782, 6014318,
    6079854, 6145390, 6210926, 6276462, 6341998, 6407534,
)

TEN = tuple(float.fromhex(h) for h in (
    "0x1.0000000000000p+0", "0x1.4248ef8fc2604p+0", "0x1.95bb8f6d46052p+0", "0x1.fec982d5bb8afp+0",
    "0x1.41857e9d4cc5fp+1", "0x1.94c583ada5b53p+1", "0x1.fd93c1f526de0p+1", "0x1.40c28430012e7p+2",
    "0x1.93d00d2348996p+2", "0x1.fc5ebcec13541p+2", "0x1.4000000000000p+3", "0x1.92db2b73b2f85p+3",
    "0x1.fb2a734897867p+3", "0x1.3f3df1c59536ep+4", "0x1.91e6de449ff77p+4", "0x1.f9f6e4990f227p+4",
    "0x1.3e7c5939384acp+5", "0x1.90f3253c017a1p+5", "0x1.f8c4106c1abfbp+5", "0x1.3dbb36138c149p+6",
    "0x1.9000000000000p+6", "0x1.f791f6509fb66p+6", "0x1.3cfa880d5eb40p+7", "0x1.8f0d6e36fa849p+7",
    "0x1.f66095d5c7f54p+7", "0x1.3c3a4edfa9759p+8", "0x1.8e1b6f87865d7p+8", "0x1.f52fee8b01d89p+8",
    "0x1.3b7a8a4390b7dp+9", "0x1.8d2a03986f19bp+9", "0x1.f400000000000p+9", "0x1.3abb39f263d20p+10",
    "0x1.8c392a10b6611p+10", "0x1.f2d0c9c4b925bp+10", "0x1.39fc5da59cf95p+11", "0x1.8b48e29793d2fp+11",
    "0x1.f1a24b6967f4cp+11", "0x1.393df516e1276p+12", "0x1.8a592cd474e5cp+12", "0x1.f074847e8ae02p+12",
    "0x1.3880000000000p+13", "0x1.896a086efcc67p+13", "0x1.ef477494e3f95p+13", "0x1.37c27e1af3b79p+14",
    "0x1.887b750f0437ap+14", "0x1.ee1b1b3d78c7ap+14", "0x1.37056f21e0f90p+15", "0x1.878d725c99713p+15",
    "0x1.ecef7809921f4p+15", "0x1.3648d2cf16cc1p+16", "0x1.86a0000000000p+16", "0x1.ebc48a8abbf81p+16",
    "0x1.358ca8dd0e7bdp+17", "0x1.85b31da1b0a57p+17", "0x1.ea9a5252c5458p+17", "0x1.34d0f1066b7ccp+18",
    "0x1.84c6caea59374p+18", "0x1.e970cef3bfcd8p+18", "0x1.3415ab05fb538p+19", "0x1.83db0782dc7f1p+19",
    "0x1.e848000000000p+19",
))


def phred(depth: int, support: int) -> int:
    """Q of one emitted character (the same 6-step search over TEN as K2q)."""
    if support <= 0:
        return 0
    e, lim = float(depth - support + 1), float(depth + 2)
    q = 0
    for step in (32, 16, 8, 4, 2, 1):
        if q + step <= QUAL_MAX and e * TEN[q + step] <= lim:
            q += step
    return q


def insertion_phred(depth: int, depth_next: int, support: int, tie: bool) -> int:
    """Q of every character of an inserted string: support = the chosen string's count in the slot's insertion dict,
    D = max(min(depth, depth_next), support) with the two ACGT depths the vote's 'I' rule compares; a tie emits "N"
    with Q0."""
    if tie:
        return 0
    return phred(max(min(depth, depth_next), support), support)
