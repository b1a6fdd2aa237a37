/* kindel_fqoracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The CPU checker of the per-base consensus qualities (an extension: the reference has no such output), in plain
 * single-threaded C, next to oracle/kindel_oracle.c.  There is no reference to pin it against: it is written as a
 * linear search over q and a sequential walk over the positions, and held against oracle/py_fqoracle.py (all 61 q at
 * once per slot, in numpy) and the product (tests/test_fastq.py).
 *
 * Q of an emitted character:  Q = 0 when the support k is 0, else the largest q in 0..60 with
 *   (double)(D - k + 1) * TEN[q] <= (double)(D + 2),  TEN[q] = the correctly rounded double of 10^(q/10).
 * A base: D = A + C + G + T; k = the called base's count (call byte bits 0-2 = 0..3), the summed counts of a multi-base
 * IUPAC set (bit 7, mask in bits 0-3, A=1 C=2 G=4 T=8) except the set of all four (the letter N), else 0.
 * An inserted string: k = its count in the position's insertion dict, D = max(min(depth, depth_next), k) with
 * depth_next the ACGT depth of the next slot (0 behind the last slot); a tie emits "N" at Q0.  A CDR patch: Q0.
 * fqoracle_fastq takes the Q of every emitted base from slot_qual[s] instead when it is not NULL (the quality vote's Q).
 */
#include <ctype.h>
#include <stdint.h>
#include <string.h>

static const double TEN[61] = {
    0x1.0000000000000p+0, 0x1.4248ef8fc2604p+0, 0x1.95bb8f6d46052p+0, 0x1.fec982d5bb8afp+0,
    0x1.41857e9d4cc5fp+1, 0x1.94c583ada5b53p+1, 0x1.fd93c1f526de0p+1, 0x1.40c28430012e7p+2,
    0x1.93d00d2348996p+2, 0x1.fc5ebcec13541p+2, 0x1.4000000000000p+3, 0x1.92db2b73b2f85p+3,
    0x1.fb2a734897867p+3, 0x1.3f3df1c59536ep+4, 0x1.91e6de449ff77p+4, 0x1.f9f6e4990f227p+4,
    0x1.3e7c5939384acp+5, 0x1.90f3253c017a1p+5, 0x1.f8c4106c1abfbp+5, 0x1.3dbb36138c149p+6,
    0x1.9000000000000p+6, 0x1.f791f6509fb66p+6, 0x1.3cfa880d5eb40p+7, 0x1.8f0d6e36fa849p+7,
    0x1.f66095d5c7f54p+7, 0x1.3c3a4edfa9759p+8, 0x1.8e1b6f87865d7p+8, 0x1.f52fee8b01d89p+8,
    0x1.3b7a8a4390b7dp+9, 0x1.8d2a03986f19bp+9, 0x1.f400000000000p+9, 0x1.3abb39f263d20p+10,
    0x1.8c392a10b6611p+10, 0x1.f2d0c9c4b925bp+10, 0x1.39fc5da59cf95p+11, 0x1.8b48e29793d2fp+11,
    0x1.f1a24b6967f4cp+11, 0x1.393df516e1276p+12, 0x1.8a592cd474e5cp+12, 0x1.f074847e8ae02p+12,
    0x1.3880000000000p+13, 0x1.896a086efcc67p+13, 0x1.ef477494e3f95p+13, 0x1.37c27e1af3b79p+14,
    0x1.887b750f0437ap+14, 0x1.ee1b1b3d78c7ap+14, 0x1.37056f21e0f90p+15, 0x1.878d725c99713p+15,
    0x1.ecef7809921f4p+15, 0x1.3648d2cf16cc1p+16, 0x1.86a0000000000p+16, 0x1.ebc48a8abbf81p+16,
    0x1.358ca8dd0e7bdp+17, 0x1.85b31da1b0a57p+17, 0x1.ea9a5252c5458p+17, 0x1.34d0f1066b7ccp+18,
    0x1.84c6caea59374p+18, 0x1.e970cef3bfcd8p+18, 0x1.3415ab05fb538p+19, 0x1.83db0782dc7f1p+19,
    0x1.e848000000000p+19,
};

int fqoracle_phred(int64_t d, int64_t k) {
    if (k <= 0) return 0;
    int q = 0;
    while (q < 60 && (double)(d - k + 1) * TEN[q + 1] <= (double)(d + 2)) ++q;
    return q;
}

static int64_t acgt(const int32_t* counts, int64_t n_slots, int64_t s) {
    int64_t d = 0;
    if (s < n_slots)
        for (int b = 0; b < 4; ++b) d += counts[(int64_t)b * n_slots + s];
    return d;
}

static int slot_q(const int32_t* counts, int64_t n_slots, int64_t s, uint8_t call) {
    int64_t k = 0;
    if (call & 0x80) {
        if ((call & 15) != 15)
            for (int b = 0; b < 4; ++b)
                if (call & (1 << b)) k += counts[(int64_t)b * n_slots + s];
    } else if ((call & 7) < 4) {
        k = counts[(int64_t)(call & 7) * n_slots + s];
    }
    return fqoracle_phred(acgt(counts, n_slots, s), k);
}

/* qual[s] for every slot of counts[>= 4][n_slots] and its call bytes */
void fqoracle_qual(const int32_t* counts, const uint8_t* calls, int64_t n_slots, uint8_t* qual) {
    for (int64_t s = 0; s < n_slots; ++s) qual[s] = (uint8_t)slot_q(counts, n_slots, s, calls[s]);
}

/* One contig (slots s0 .. s0 + L) walked position by position as the reference's consensus_sequence does
 * (kindel/kindel.py:387-430), writing the text and the Phred+33 qualities side by side.  Per position p:
 *   ins_k[p]    count of the modal inserted string (-1: a tie), read where the call has change 'I'
 *   ins_off[p .. p+1]  that string (as counted, upper case) in ins_bytes
 *   patch_skip[p]  INT64_MIN: no CDR patch starts here; else the patch (patch_off / patch_bytes) and end - start - 1
 * slot_qual: NULL (the Q of slot_q), or the Q of every slot's emitted base.
 * Returns the length written to text / qual (both at least the untrimmed length). */
int64_t fqoracle_fastq(const int32_t* counts, int64_t n_slots, int64_t s0, int64_t L, const uint8_t* calls,
                       const int64_t* ins_k, const int64_t* ins_off, const char* ins_bytes, const int64_t* patch_skip,
                       const int64_t* patch_off, const char* patch_bytes, const uint8_t* slot_qual, int trim_ends,
                       int uppercase, char* text, char* qual) {
    static const char* iupac = "=ACMGRSVTWYHKDBN";
    static const char* acgtn = "ACGTN";
    int64_t n = 0, skip = 0;
    for (int64_t p = 0; p < L; ++p) {
        if (skip != 0) { /* a negative count never returns to 0: nothing more is emitted */
            --skip;
            continue;
        }
        if (patch_skip[p] != INT64_MIN) {
            for (int64_t j = patch_off[p]; j < patch_off[p + 1]; ++j) {
                text[n] = (char)tolower((unsigned char)patch_bytes[j]);
                qual[n++] = '!';
            }
            skip = patch_skip[p];
            continue;
        }
        const int64_t s = s0 + p;
        const uint8_t c = calls[s];
        const int change = (c >> 4) & 3;
        if (change == 1) continue; /* 'D' */
        if (change == 3) {
            if (ins_k[p] < 0) {
                text[n] = 'N';
                qual[n++] = '!';
            } else {
                const int64_t d = acgt(counts, n_slots, s), dn = acgt(counts, n_slots, s + 1);
                int64_t D = d < dn ? d : dn;
                if (ins_k[p] > D) D = ins_k[p];
                const char qc = (char)(33 + fqoracle_phred(D, ins_k[p]));
                for (int64_t j = ins_off[p]; j < ins_off[p + 1]; ++j) {
                    text[n] = (char)tolower((unsigned char)ins_bytes[j]);
                    qual[n++] = qc;
                }
            }
        }
        text[n] = (c & 0x80) ? iupac[c & 15] : acgtn[(c & 7) > 4 ? 4 : (c & 7)];
        qual[n++] = (char)(33 + (slot_qual ? slot_qual[s] : slot_q(counts, n_slots, s, c)));
    }
    int64_t a = 0, b = n;
    if (trim_ends) {
        while (a < b && text[a] == 'N') ++a;
        while (b > a && text[b - 1] == 'N') --b;
        memmove(text, text + a, (size_t)(b - a));
        memmove(qual, qual + a, (size_t)(b - a));
    }
    if (uppercase)
        for (int64_t j = 0; j < b - a; ++j) text[j] = (char)toupper((unsigned char)text[j]);
    return b - a;
}
