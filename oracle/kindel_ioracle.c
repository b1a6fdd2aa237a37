/* kindel_ioracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The CPU checker of the IUPAC vote (an extension: the reference has no such option), in plain single-threaded C,
 * next to oracle/kindel_oracle.c.  There is no reference to pin it against: it is written in the set / level form of
 * the definition and held against oracle/py_ioracle.py, an independent loop over tie groups (tests/test_iupac.py).
 *
 * calls[s] for every slot s of counts[19][n_slots] (columns 0-4 A,C,G,T,N, 5 deletions, 6 insertions):
 *   the reference's decisions (kindel/kindel.py:402-424), with depth = A + C + G + T and depth_next that of slot s+1
 *   (0 behind the last slot):  2 del > depth -> 'D' (0x14);  depth < ceil(min_depth) -> 'N' (0x24);  else the change
 *   is 'I' (3) when 2 ins > min(depth, depth_next), none (0) otherwise, and the base is the IUPAC vote's:
 *     depth == 0 -> N (code 4).  Else for each base b with count(b) > 0, L(b) = the sum of the counts of all bases with
 *     count >= count(b); v = the largest count(b) with (double)L(b) >= t * (double)depth; S = {b : count(b) >= v}.
 *     |S| == 1: change << 4 | the base's code (A,C,G,T = 0..3); |S| >= 2: 0x80 | change << 4 | mask (A=1 C=2 G=4 T=8).
 */
#include <stdint.h>

void ioracle_vote(const int32_t* counts, int64_t n_slots, int64_t min_depth_ceil, double t, uint8_t* calls) {
    for (int64_t s = 0; s < n_slots; ++s) {
        int64_t w[4], depth = 0, depth_next = 0;
        for (int k = 0; k < 4; ++k) {
            w[k] = counts[(int64_t)k * n_slots + s];
            depth += w[k];
            if (s + 1 < n_slots) depth_next += counts[(int64_t)k * n_slots + s + 1];
        }
        const int64_t del = counts[(int64_t)5 * n_slots + s], ins = counts[(int64_t)6 * n_slots + s];
        if (2 * del > depth) {
            calls[s] = (1 << 4) | 4;
            continue;
        }
        if (depth < min_depth_ceil) {
            calls[s] = (2 << 4) | 4;
            continue;
        }
        const int change = 2 * ins > (depth < depth_next ? depth : depth_next) ? 3 : 0;
        if (depth == 0) {
            calls[s] = (uint8_t)((change << 4) | 4);
            continue;
        }
        int64_t v = -1;
        for (int b = 0; b < 4; ++b) {
            if (w[b] <= 0) continue;
            int64_t level = 0; /* L(b) */
            for (int k = 0; k < 4; ++k)
                if (w[k] >= w[b]) level += w[k];
            if ((double)level >= t * (double)depth && w[b] > v) v = w[b];
        }
        int mask = 0, n = 0, only = 0;
        for (int b = 0; b < 4; ++b)
            if (w[b] >= v) {
                mask |= 1 << b;
                n += 1;
                only = b;
            }
        calls[s] = (uint8_t)(n == 1 ? (change << 4) | only : 0x80 | (change << 4) | mask);
    }
}
