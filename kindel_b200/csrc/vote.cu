// vote.cu -- K2: per-position majority vote (or, as an extension, the IUPAC vote); K2d: derived depth columns;
// K2p: fused cross-GPU count reduction + vote over NVLink peer memory.
//
// K2 restates, for every table slot at once, the body of consensus_sequence
// (kindel/kindel.py:402-424) with consensus() (kindel.py:369-381) inlined.  It is a pure streaming
// kernel: 7 int32 columns in (28 B/slot), one call byte out; each thread owns 4 consecutive slots
// (128-bit loads per column, one 32-bit store), the look-ahead depth `aligned_depth_next`
// (kindel.py:405-410) comes from the neighbouring lane by shuffle, the last lane of a warp reads
// it.  Slot ref_len of every contig holds zero in the weight columns, which is exactly the
// reference's `except IndexError: aligned_depth_next = 0` at the last position, so the kernel
// needs no contig table.
#include "kdl_common.cuh"

namespace kdl {

struct Peers {
    const int32_t* tab[16];
    long long lo[16], hi[16];  // footprint of each table: zero outside [lo, hi)
    int n;
};

template <bool kPeers>
__device__ __forceinline__ int4 load4(const int32_t* __restrict__ counts, const Peers& peers, int col,
                                      long long n_slots, long long s) {
    if constexpr (!kPeers) {
        return __ldg(reinterpret_cast<const int4*>(counts + (long long)col * n_slots + s));
    } else {
        int4 acc = make_int4(0, 0, 0, 0);
        for (int p = 0; p < peers.n; ++p) {
            if (s + 4 <= peers.lo[p] || s >= peers.hi[p]) continue;  // nothing of peer p here
            // peer tables are written by other GPUs: plain (coherent) loads, not the nc path
            const int4 v = *reinterpret_cast<const int4*>(peers.tab[p] + (long long)col * n_slots + s);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        return acc;
    }
}

template <bool kPeers>
__device__ __forceinline__ int load1(const int32_t* __restrict__ counts, const Peers& peers, int col,
                                     long long n_slots, long long s) {
    if constexpr (!kPeers) {
        return __ldg(counts + (long long)col * n_slots + s);
    } else {
        int acc = 0;
        for (int p = 0; p < peers.n; ++p)
            if (s >= peers.lo[p] && s < peers.hi[p]) acc += peers.tab[p][(long long)col * n_slots + s];
        return acc;
    }
}

// n_slots % 4 == 0, slot_lo % 4 == 0.  One thread = 4 slots.  Vote: MajorityVote (the reference's), IupacVote or
// QualityVote (kdl_common.cuh); the policy argument comes last and defaults to the majority, so the majority
// instantiations keep their code and their callers.
template <bool kPeers, class Vote = MajorityVote>
__global__ void __launch_bounds__(256)
vote_kernel(const int32_t* __restrict__ counts, Peers peers, long long n_slots, long long slot_lo,
            long long slot_hi, long long min_depth_ceil, uint8_t* __restrict__ calls,
            int32_t* __restrict__ reduced, Vote vote = Vote()) {
    const long long quad = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long s = slot_lo + quad * 4;
    const bool active = s < slot_hi;
    int4 v[KDL_NVOTE_COL];
    long long d0 = 0;
    if (active) {
#pragma unroll
        for (int k = 0; k < KDL_NVOTE_COL; ++k) v[k] = load4<kPeers>(counts, peers, k, n_slots, s);
        d0 = (long long)v[0].x + v[1].x + v[2].x + v[3].x;
        if constexpr (kPeers) {
            if (reduced) {
#pragma unroll
                for (int k = 0; k < KDL_NVOTE_COL; ++k)
                    *reinterpret_cast<int4*>(reduced + (long long)k * n_slots + s) = v[k];
            }
        }
    }
    // depth of slot s+4 = first slot of the next lane's quad
    long long dn = __shfl_down_sync(0xffffffffu, d0, 1);
    if ((threadIdx.x & 31) == 31 || !active || s + 4 >= slot_hi) {
        dn = 0;
        if (active && s + 4 < n_slots) {
#pragma unroll
            for (int k = 0; k < 4; ++k) dn += load1<kPeers>(counts, peers, k, n_slots, s + 4);
        }
    }
    if (!active) return;
    const long long d1 = (long long)v[0].y + v[1].y + v[2].y + v[3].y;
    const long long d2 = (long long)v[0].z + v[1].z + v[2].z + v[3].z;
    const long long d3 = (long long)v[0].w + v[1].w + v[2].w + v[3].w;
    const unsigned c0 = vote(s, v[0].x, v[1].x, v[2].x, v[3].x, v[4].x, v[5].x, v[6].x, d1, min_depth_ceil);
    const unsigned c1 = vote(s + 1, v[0].y, v[1].y, v[2].y, v[3].y, v[4].y, v[5].y, v[6].y, d2, min_depth_ceil);
    const unsigned c2 = vote(s + 2, v[0].z, v[1].z, v[2].z, v[3].z, v[4].z, v[5].z, v[6].z, d3, min_depth_ceil);
    const unsigned c3 = vote(s + 3, v[0].w, v[1].w, v[2].w, v[3].w, v[4].w, v[5].w, v[6].w, dn, min_depth_ceil);
    *reinterpret_cast<uint32_t*>(calls + s) = c0 | (c1 << 8) | (c2 << 16) | (c3 << 24);
}

// ---- K2x / K2g: the exchange without NCCL (flags + reduce + vote, then a pull of the call bytes) --
struct Exchange {
    Peers peers;
    uint8_t* calls[16];
    long long slice_lo[16], slice_hi[16];
    int32_t* ready[16];     // ready[p]: flag array living in rank p's block
    int32_t* done[16];
    int32_t* ready_local;   // = ready[rank]: written by the peers
    int32_t* done_local;
    int32_t* counter;
    int rank;
};

#ifndef KDL_HOST_EMU
__device__ __forceinline__ int ld_acquire_sys(const int32_t* p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(int32_t* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#endif  // KDL_HOST_EMU (tests/emu/ supplies stand-ins)

// "my table is complete": runs after the pileup kernels in stream order
__global__ void exchange_signal_kernel(Exchange x, int epoch) {
    const int p = threadIdx.x;
    __threadfence_system();
    if (p < x.peers.n) st_release_sys(x.ready[p] + x.rank, epoch);
}

// K2g: one CTA group per peer pulls that peer's call slice once the peer has published it
__global__ void __launch_bounds__(256) exchange_gather_kernel(Exchange x, int epoch) {
    const int p = blockIdx.y;
    if (p == x.rank) return;
    if (threadIdx.x == 0)
        while (ld_acquire_sys(x.done_local + p) < epoch) __nanosleep(32);
    __syncthreads();
    // the peer's slice [lo, hi) (multiples of 4): 16-byte vector copies over its 16-aligned middle, bytes at the rims
    const long long lo = x.slice_lo[p], hi = x.slice_hi[p];
    long long a16 = (lo + 15) & ~15ll, b16 = hi & ~15ll;
    if (a16 > b16) a16 = b16 = hi;  // (a slice shorter than one vector: bytes only; lo..hi below)
    const long long n16 = (b16 - a16) >> 4;
    const uint4* src = reinterpret_cast<const uint4*>(x.calls[p] + a16);
    uint4* dst = reinterpret_cast<uint4*>(x.calls[x.rank] + a16);
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; v + 3 * stride < n16; v += 4 * stride) {  // four NVLink reads in flight per thread
        const uint4 a0 = src[v], a1 = src[v + stride], a2 = src[v + 2 * stride], a3 = src[v + 3 * stride];
        dst[v] = a0; dst[v + stride] = a1; dst[v + 2 * stride] = a2; dst[v + 3 * stride] = a3;
    }
    for (; v < n16; v += stride) dst[v] = src[v];
    if (blockIdx.x == 0) {
        const long long head_end = a16 < hi ? a16 : hi;
        for (long long s = lo + threadIdx.x; s < head_end; s += blockDim.x) x.calls[x.rank][s] = x.calls[p][s];
        for (long long s = (b16 > head_end ? b16 : head_end) + threadIdx.x; s < hi; s += blockDim.x) x.calls[x.rank][s] = x.calls[p][s];
    }
}

template <class Vote = MajorityVote>
__global__ void __launch_bounds__(256)
vote_exchange_kernel(Exchange x, long long n_slots, long long min_depth_ceil, int epoch, Vote vote = Vote()) {
    // this kernel runs after the rank's pileup kernels in stream order, so its own table is complete:
    // CTA 0 publishes that to every peer (kdl_exchange_signal is then optional) ...
    if (blockIdx.x == 0 && threadIdx.x < x.peers.n) {
        __threadfence_system();
        st_release_sys(x.ready[threadIdx.x] + x.rank, epoch);
    }
    const Peers& peers = x.peers;
    const long long slot_lo = x.slice_lo[x.rank], slot_hi = x.slice_hi[x.rank];
    const long long quads = (slot_hi - slot_lo + 3) >> 2;
    const long long per_cta = (((quads + gridDim.x - 1) / gridDim.x) + 31) & ~31ll;  // whole warps iterate together
    const long long q0 = (long long)blockIdx.x * per_cta;
    long long q1 = q0 + per_cta;
    if (q1 > ((quads + 31) & ~31ll)) q1 = (quads + 31) & ~31ll;
    // ... and every table this CTA reads must be complete: ready[rank][p] >= epoch for the peers p whose footprint
    // overlaps the chunk (the look-ahead depth reads up to 4 slots past it)
    __shared__ unsigned overlap_mask;
    if (threadIdx.x == 0) overlap_mask = 0u;
    __syncthreads();
    if (threadIdx.x < peers.n && q0 < q1) {
        const int p = threadIdx.x;
        const long long c_lo = slot_lo + q0 * 4, c_hi = slot_lo + q1 * 4 + 4;
        if (peers.lo[p] < c_hi && peers.hi[p] > c_lo) {
            atomicOr(&overlap_mask, 1u << p);
            if (p != x.rank)
                while (ld_acquire_sys(x.ready_local + p) < epoch) __nanosleep(32);
        }
    }
    __syncthreads();
    const unsigned mask = overlap_mask;
    uint8_t* __restrict__ calls = x.calls[x.rank];
    for (long long quad = q0 + threadIdx.x; quad < q1; quad += blockDim.x) {
        const long long s = slot_lo + quad * 4;
        const bool active = s < slot_hi;
        int4 v[KDL_NVOTE_COL];
        long long d0 = 0;
        if (active) {
#pragma unroll
            for (int k = 0; k < KDL_NVOTE_COL; ++k) v[k] = make_int4(0, 0, 0, 0);
            for (unsigned m = mask; m; m &= m - 1) {
                const int p = __ffs(m) - 1;
                if (s + 4 <= peers.lo[p] || s >= peers.hi[p]) continue;  // nothing of table p here
                int4 t[KDL_NVOTE_COL];  // seven independent 128-bit loads in flight per table
#pragma unroll
                for (int k = 0; k < KDL_NVOTE_COL; ++k)
                    t[k] = *reinterpret_cast<const int4*>(peers.tab[p] + (long long)k * n_slots + s);
#pragma unroll
                for (int k = 0; k < KDL_NVOTE_COL; ++k) {
                    v[k].x += t[k].x; v[k].y += t[k].y; v[k].z += t[k].z; v[k].w += t[k].w;
                }
            }
            d0 = (long long)v[0].x + v[1].x + v[2].x + v[3].x;
        }
        long long dn = __shfl_down_sync(0xffffffffu, d0, 1);
        if ((threadIdx.x & 31) == 31 || !active || s + 4 >= slot_hi) {
            dn = 0;
            if (active && s + 4 < n_slots) {
                for (unsigned m = mask; m; m &= m - 1) {
                    const int p = __ffs(m) - 1;
                    if (s + 4 >= peers.lo[p] && s + 4 < peers.hi[p]) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) dn += peers.tab[p][(long long)k * n_slots + s + 4];
                    }
                }
            }
        }
        if (active) {
            const long long d1 = (long long)v[0].y + v[1].y + v[2].y + v[3].y;
            const long long d2 = (long long)v[0].z + v[1].z + v[2].z + v[3].z;
            const long long d3 = (long long)v[0].w + v[1].w + v[2].w + v[3].w;
            const unsigned c0 = vote(s, v[0].x, v[1].x, v[2].x, v[3].x, v[4].x, v[5].x, v[6].x, d1, min_depth_ceil);
            const unsigned c1 = vote(s + 1, v[0].y, v[1].y, v[2].y, v[3].y, v[4].y, v[5].y, v[6].y, d2, min_depth_ceil);
            const unsigned c2 = vote(s + 2, v[0].z, v[1].z, v[2].z, v[3].z, v[4].z, v[5].z, v[6].z, d3, min_depth_ceil);
            const unsigned c3 = vote(s + 3, v[0].w, v[1].w, v[2].w, v[3].w, v[4].w, v[5].w, v[6].w, dn, min_depth_ceil);
            *reinterpret_cast<uint32_t*>(calls + s) = c0 | (c1 << 8) | (c2 << 16) | (c3 << 24);
        }
    }
    // last CTA out publishes "my slice is voted (and I no longer read your tables)" to every peer
    __syncthreads();
    __shared__ int last;
    if (threadIdx.x == 0) {
        __threadfence();
        last = (atomicAdd(x.counter, 1) == (int)gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        if (threadIdx.x == 0) *x.counter = 0;
        __threadfence_system();
        if (threadIdx.x < peers.n) st_release_sys(x.done[threadIdx.x] + x.rank, epoch);
    }
}

// Derived columns (kindel/kindel.py:83-96, :450): out[5][n_slots].
__global__ void __launch_bounds__(256)
derive_kernel(const int32_t* __restrict__ counts, long long n_slots, int32_t* __restrict__ out) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    int w[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) w[k] = __ldg(counts + (long long)k * n_slots + s);
    int freq, raw;
    base_vote(w[0], w[1], w[2], w[3], w[4], &freq, &raw);
    int csd = 0, ced = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        csd += __ldg(counts + (long long)(KDL_CSW_A + k) * n_slots + s);
        ced += __ldg(counts + (long long)(KDL_CEW_A + k) * n_slots + s);
    }
    out[0 * n_slots + s] = freq;  // aligned_depth - discordant_depth (kindel.py:84-89)
    out[1 * n_slots + s] = csd;
    out[2 * n_slots + s] = ced;
    out[3 * n_slots + s] = csd + ced;
    out[4 * n_slots + s] = w[0] + w[1] + w[2] + w[3];
}

template __global__ void vote_kernel<false>(const int32_t*, Peers, long long, long long, long long,
                                            long long, uint8_t*, int32_t*, MajorityVote);
template __global__ void vote_kernel<true>(const int32_t*, Peers, long long, long long, long long,
                                           long long, uint8_t*, int32_t*, MajorityVote);
template __global__ void vote_kernel<false, IupacVote>(const int32_t*, Peers, long long, long long, long long,
                                                       long long, uint8_t*, int32_t*, IupacVote);
template __global__ void vote_kernel<false, QualityVote>(const int32_t*, Peers, long long, long long, long long,
                                                         long long, uint8_t*, int32_t*, QualityVote);
template __global__ void vote_exchange_kernel<MajorityVote>(Exchange, long long, long long, int, MajorityVote);
template __global__ void vote_exchange_kernel<IupacVote>(Exchange, long long, long long, int, IupacVote);

}  // namespace kdl
