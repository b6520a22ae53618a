// Multi-stream SHA-256 for sm_90a: one independent message per lane, a warp hashes 32
// messages in lock step.  This is the kernel behind every digest modelx-b200 produces:
//   - leaf / chunk / upper tree levels of a blob (uniform segments of one buffer),
//   - batches of whole blobs (arbitrary spans; the reference's one-digest-per-file semantics,
//     pkg/client/push.go:149-161 and pull.go:115-123, across many files at once),
//   - chained segments of a single stream (hash.Hash-shaped incremental API, helper.go:46).
// Pure 32-bit integer work, no tensor cores.  In the throughput kernel (k_sha256_lanes) the 16-word schedule
// and the chain state live in registers and round constants are instruction immediates (no shared memory);
// the latency kernel for few long chains (k_sha256_chains_coop) passes W+K between two warps through 16 KB
// of shared memory.
#include "kernels.h"
#include "sha256_device.cuh"
#include <atomic>
#include <cstdlib>
#include <cstdio>
#include <vector>

namespace mxd {

namespace {

// 64-thread CTAs: the finer work quantum per CTA (1 MiB of leaves).
constexpr int kThreads = 64;

__device__ __forceinline__ uint4 ldg128(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// 64 message bytes at p (any alignment) -> 16 big-endian words.
// a = p & 3; q = p - a is 4-byte aligned.  Little-endian word k of the block is
// funnelshift_r(q[k], q[k+1], 8a).  q[16] is only touched when a != 0, in which case it holds
// the block's last byte(s), so it is inside the message.
__device__ __forceinline__ void load_block_unaligned(const uint8_t* p, uint32_t (&w)[16]) {
    const uint32_t a = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p - a);
    if (a == 0) {
#pragma unroll
        for (int k = 0; k < 16; ++k) w[k] = bswap32(__ldg(q + k));
    } else {
        uint32_t lo = __ldg(q);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            uint32_t hi = __ldg(q + k + 1);
            w[k] = bswap32(__funnelshift_r(lo, hi, 8 * a));
            lo = hi;
        }
    }
}

__device__ __forceinline__ void unpack_block(const uint4& v0, const uint4& v1, const uint4& v2, const uint4& v3,
                                             uint32_t (&w)[16]) {
    w[0] = bswap32(v0.x);  w[1] = bswap32(v0.y);  w[2] = bswap32(v0.z);  w[3] = bswap32(v0.w);
    w[4] = bswap32(v1.x);  w[5] = bswap32(v1.y);  w[6] = bswap32(v1.z);  w[7] = bswap32(v1.w);
    w[8] = bswap32(v2.x);  w[9] = bswap32(v2.y);  w[10] = bswap32(v2.z); w[11] = bswap32(v2.w);
    w[12] = bswap32(v3.x); w[13] = bswap32(v3.y); w[14] = bswap32(v3.z); w[15] = bswap32(v3.w);
}

// Where message m of a launch lives and what to do with it (shared by both SHA-256 kernels).
struct Located {
    const uint8_t* ptr; uint64_t len, prefix;
    uint32_t sidx, oidx;      // chain-state slot / digest slot
    int fin; bool live, load_state;
};
__device__ __forceinline__ Located locate(const MsgJob& j, uint64_t m) {
    Located L;
    L.ptr = nullptr; L.len = 0; L.prefix = j.prefix_all; L.sidx = (uint32_t)m; L.oidx = (uint32_t)m;
    L.fin = j.finalize; L.live = m < j.nmsg; L.load_state = false;
    if (!L.live) return L;
    if (j.descs != nullptr) {
        const LaneDesc d = j.descs[m];
        L.ptr = static_cast<const uint8_t*>(d.ptr); L.len = d.len; L.prefix = d.prefix;
        L.sidx = d.lane; L.oidx = d.oidx;
        L.fin = (d.ctl & kFinalize) != 0; L.live = (d.ctl & kSkip) == 0;
        L.load_state = L.live && (d.ctl & kFresh) == 0;
    } else if (j.base != nullptr) {
        const uint64_t off = m * j.seg;
        L.ptr = j.base + off;
        L.len = (off < j.nbytes) ? ((j.nbytes - off < j.seg) ? j.nbytes - off : j.seg) : 0;
        L.load_state = j.state != nullptr;
    } else {
        const DevSpan sp = reinterpret_cast<const DevSpan*>(j.spans)[m];
        L.ptr = static_cast<const uint8_t*>(sp.ptr);
        L.len = sp.len;
        L.load_state = j.state != nullptr;
    }
    return L;
}

// Run one lane's chain over its message: `nfull` full blocks at ptr, then (nblk > nfull) the padded tail block and,
// if needed, the length block.  All 32 lanes of the warp must call this together.
__device__ __forceinline__ void absorb(const uint8_t* ptr, const uint64_t nfull, const uint32_t r, const uint64_t nblk,
                                       const uint64_t bits, const bool live, uint32_t (&h)[8], const uint32_t one) {
    // Hot loop: when every lane of the warp has a 16-byte aligned message (always true for tree
    // levels) the full blocks run in a straight-line loop of their own: 4 x LDG.128 per block, the
    // next block prefetched into registers while this one is compressed.  Keeping this loop free of
    // control-flow merges matters: after a merge ptxas must wait for every load that any incoming
    // path may have in flight, which would serialise the prefetch with the compress.
    // Lane i streams its own message, so a request touches 32 different lines but consumes whole
    // 32-byte sectors: DRAM traffic equals the algorithmic bytes.
    const bool warp_aligned = __all_sync(0xffffffffu, (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0);
    uint32_t w[16];
    uint64_t b = 0;
    if (warp_aligned && live && nfull) {
        const uint4* p4 = reinterpret_cast<const uint4*>(ptr);
        uint4 v0 = ldg128(p4), v1 = ldg128(p4 + 1), v2 = ldg128(p4 + 2), v3 = ldg128(p4 + 3);
        for (; b < nfull; ++b) {
            unpack_block(v0, v1, v2, v3, w);
            p4 += (b + 1 < nfull) ? 4 : 0;   // last iteration re-reads its own block (L1 hit) instead of branching
            v0 = ldg128(p4); v1 = ldg128(p4 + 1); v2 = ldg128(p4 + 2); v3 = ldg128(p4 + 3);
            sha256_compress(h, w, one);
        }
    }
    // Everything else: unaligned full blocks, the padded tail block and the length block.
    for (; b < nblk; ++b) {
        if (b < nfull) {
            load_block_unaligned(ptr + (b << 6), w);
        } else if (b == nfull) {
            // r tail bytes, the 0x80 marker, zeros; the length too when it fits (r < 56)
            const uint8_t* t = ptr + (nfull << 6);
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                uint32_t word = 0;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint32_t idx = 4 * k + q;
                    if (idx < r) word |= (uint32_t)__ldg(t + idx) << (24 - 8 * q);
                    else if (idx == r) word |= 0x80u << (24 - 8 * q);
                }
                w[k] = word;
            }
            if (r < 56) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
        } else {
#pragma unroll
            for (int k = 0; k < 14; ++k) w[k] = 0;
            w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
        }
        sha256_compress(h, w, one);
    }

}

// MINB = resident CTAs per SM the register allocator must allow (12 x 64 threads -> 80 registers, 16 -> 63).
// THREADS: 64, or 32 (MXD_TUNE_CTA=32: one warp per CTA, 24 CTAs per SM -- a finer completion quantum for the drain).
template <int MINB, int THREADS = kThreads>
__global__ void __launch_bounds__(THREADS, MINB) k_sha256_lanes(const MsgJob j) {
    const uint64_t m = (uint64_t)blockIdx.x * THREADS + threadIdx.x;
    const uint32_t one = j.one;
    const Located L = locate(j, m);
    const uint8_t* ptr = L.ptr;
    const uint64_t len = L.len;
    const bool live = L.live;
    const int fin = L.fin;
    uint32_t h[8];
    if (L.load_state) {
#pragma unroll
        for (int i = 0; i < 8; ++i) h[i] = j.state[8 * (uint64_t)L.sidx + i];
    } else {
        sha256_iv(h);
    }
    const uint64_t nfull = len >> 6;
    const uint32_t r = (uint32_t)(len & 63u);
    // blocks this lane compresses: the full ones, then (when finalizing) the padded tail block
    // and, if the 64-bit length does not fit behind the tail, one more (FIPS 180-4 section 5.1.1).
    const uint64_t nblk = live ? nfull + (fin ? (r >= 56 ? 2u : 1u) : 0u) : 0;
    const uint64_t bits = (L.prefix + len) << 3;

    absorb(ptr, nfull, r, nblk, bits, live, h, one);

    if (!live) return;
    if (!fin) {
#pragma unroll
        for (int i = 0; i < 8; ++i) j.state[8 * (uint64_t)L.sidx + i] = h[i];
        return;
    }
    uint4 lo, hi;
    lo.x = bswap32(h[0]); lo.y = bswap32(h[1]); lo.z = bswap32(h[2]); lo.w = bswap32(h[3]);
    hi.x = bswap32(h[4]); hi.y = bswap32(h[5]); hi.z = bswap32(h[6]); hi.w = bswap32(h[7]);
    uint4* o = reinterpret_cast<uint4*>(j.out + 32 * (uint64_t)L.oidx);
    o[0] = lo; o[1] = hi;
}

// =====================================================================================================
// k_sha256_chains_coop: few, long chains.  A SHA-256 chain is serial, so when a launch has only a few
// thousand messages (a push/pull of a few hundred files, one streamed file, a ring slot) the lanes
// kernel above is latency bound: a lone warp needs thousands of clk per block because the 480-instruction
// message schedule and the loads sit in the same instruction stream as the 64 dependent rounds.
// Here every 32 chains get two warps on two different SM sub-partitions:
//   warp 1 (producer)  loads/pads block b of its 32 messages (next block prefetched into registers), expands
//                      the schedule and stores W[t]+K[t] (t = 0..63) to shared memory, one stage ahead;
//   warp 0 (chain)     runs only the 64 rounds, reading W[t]+K[t] with LDS.128 (16 per block), with the
//                      round written so that a single addition follows Sigma1 on the e-chain.
// Same MsgJob contract as the lanes kernel
// (spans or segments, chained state, per-message control bytes), same results bit for bit.
// =====================================================================================================
// The producer warp of the two cooperative kernels below: loads / pads block b of its lane's message (next block
// prefetched into registers), expands the schedule and publishes W[t]+K[t] (t = 0..63) one stage ahead.
// wk element (stage, t/4, lane) lives at wk[(stage * 16 + t/4) * COLS + lane]; lanes with publish == false compute
// along (they shadow a live lane) and store nothing.
constexpr int kCoopStages = 2;                     // blocks the producer may run ahead
constexpr int kFull0 = 1, kEmpty0 = 1 + kCoopStages;   // named barrier ids (0 is __syncthreads)

__device__ __forceinline__ uint32_t mad_lo(uint32_t a, uint32_t b, uint32_t c) {        // a*b+c on the FMA pipe
    uint32_t d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" :: "r"(id), "r"(nthreads) : "memory"); }

template <int COLS>
__device__ __forceinline__ void coop_produce(uint4* wk, const int lane, const bool publish, const Located& L, const uint64_t nfull,
                                             const uint32_t r, const uint64_t nblk, const uint64_t bits, const uint64_t nmax,
                                             const uint32_t one) {
    const uint8_t* ptr = L.ptr;
    // ---------------- producer: load / pad, expand, publish W+K ---------------------------------
    // expands w[16] to the 64 schedule words, adds the round constants and publishes them for `lane`
    auto expand_store = [&](uint32_t (&w)[16], int st) {
        constexpr K256Table K = k256_table();
#pragma unroll
        for (int g = 0; g < 16; ++g) {
            uint32_t o4[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int t = 4 * g + q;
                if (t >= 16) {
                    uint32_t x = add_fma(w[t & 15], small_sigma0(w[(t + 1) & 15]), one);
                    x = add_fma(x, w[(t + 9) & 15], one);
                    w[t & 15] = add_fma(x, small_sigma1(w[(t + 14) & 15]), one);
                }
                o4[q] = add_fma(w[t & 15], K.v[t], one);
            }
            if (publish) wk[(st * 16 + g) * COLS + lane] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
    };
    const bool warp_aligned = __all_sync(0xffffffffu, (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0);
    uint32_t w[16];
    uint64_t b = 0;
    if (warp_aligned) {
        // Hot loop (aligned messages): the next block is prefetched into registers while this one is expanded,
        // so the chain warp never waits for DRAM.  Runs while ANY lane still has full blocks; lanes that ran
        // out keep re-reading their last block (or nothing) and publish nothing.
        // Lanes without a message (tail of the batch, finished files) shadow a live lane so that they do not
        // force the whole warp onto the slow path: same address, same trip count, nothing of theirs is consumed.
        const unsigned have = __ballot_sync(0xffffffffu, nblk > 0 && nfull > 0);
        const int src = have ? (__ffs(have) - 1) : 0;
        const uint64_t src_ptr = __shfl_sync(0xffffffffu, reinterpret_cast<uint64_t>(ptr), src);
        const uint64_t src_nfull = __shfl_sync(0xffffffffu, nfull, src);
        const bool shadow = (nblk == 0);      // only lanes the chain warp will never read for
        const uint8_t* hot_ptr = shadow ? reinterpret_cast<const uint8_t*>(src_ptr) : ptr;
        const uint64_t hot_nfull = shadow ? src_nfull : nfull;
        uint64_t nfull_min = have ? hot_nfull : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const uint64_t other = __shfl_xor_sync(0xffffffffu, nfull_min, o); nfull_min = other < nfull_min ? other : nfull_min; }
        if (nfull_min > 0) {
            const uint4* p4 = reinterpret_cast<const uint4*>(hot_ptr);
            uint4 v0 = ldg128(p4), v1 = ldg128(p4 + 1), v2 = ldg128(p4 + 2), v3 = ldg128(p4 + 3);
            for (; b < nfull_min; ++b) {          // every lane has a full block b here: no divergence, no merges
                const int st = (int)(b % kCoopStages);
                if (b >= (uint64_t)kCoopStages) named_bar_sync(kEmpty0 + st, 64);
                unpack_block(v0, v1, v2, v3, w);
                p4 += (b + 1 < hot_nfull) ? 4 : 0;
                v0 = ldg128(p4); v1 = ldg128(p4 + 1); v2 = ldg128(p4 + 2); v3 = ldg128(p4 + 3);
                expand_store(w, st);
                named_bar_arrive(kFull0 + st, 64);
            }
        }
    }
    // Everything else: ragged tails of the batch, unaligned messages, padding and length blocks.
    for (; b < nmax; ++b) {
        const int st = (int)(b % kCoopStages);
        if (b >= (uint64_t)kCoopStages) named_bar_sync(kEmpty0 + st, 64);   // chain warp has drained this stage
        if (b < nblk) {
            if (b < nfull) {
                load_block_unaligned(ptr + (b << 6), w);
            } else if (b == nfull) {
                const uint8_t* t = ptr + (nfull << 6);
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    uint32_t word = 0;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t idx = 4 * k + q;
                        if (idx < r) word |= (uint32_t)__ldg(t + idx) << (24 - 8 * q);
                        else if (idx == r) word |= 0x80u << (24 - 8 * q);
                    }
                    w[k] = word;
                }
                if (r < 56) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
            } else {
#pragma unroll
                for (int k = 0; k < 14; ++k) w[k] = 0;
                w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
            }
            expand_store(w, st);
        }
        named_bar_arrive(kFull0 + st, 64);
    }
}

// VARIANT: how the chain warp writes one round (same arithmetic, different dependency shape; MXD_TUNE_CHAIN selects):
//   0  one addition behind Sigma1 on the e-chain, T1 shared by both outputs                     (round 1's choice)
//   1  the textbook form: T1 = h+K+W+Ch+Sigma1, e' = d+T1, a' = T1+Sigma0+Maj (6 additions)
//   2  d pre-added: x = (W+K+h)+d is ready before e is, e' = (x+Ch)+Sigma1, T1 = e'-d; the e-chain is
//      SHF -> LOP3 -> IMAD = 13 clk instead of 17, so the round is bound by the ALU pipe (20 clk), not by latency
template <int VARIANT>
__global__ void __launch_bounds__(64) k_sha256_chains_coop(const MsgJob j) {
    // wk[stage][t/4][lane] = {W+K for rounds 4g..4g+3} of that lane's current block
    __shared__ uint4 wk[kCoopStages][16][32];
    const int lane = threadIdx.x & 31;
    const int role = threadIdx.x >> 5;            // 0 = chain warp, 1 = producer warp
    const uint64_t m = (uint64_t)blockIdx.x * 32 + lane;
    const uint32_t one = j.one;
    const Located L = locate(j, m);
    const uint64_t len = L.len;
    const bool live = L.live;
    const int fin = L.fin;
    const uint64_t nfull = len >> 6;
    const uint32_t r = (uint32_t)(len & 63u);
    const uint64_t nblk = live ? nfull + (fin ? (r >= 56 ? 2u : 1u) : 0u) : 0;
    const uint64_t bits = (L.prefix + len) << 3;
    // both warps iterate to the longest chain of the 32; shorter lanes idle through the barriers
    uint64_t nmax = nblk;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const uint64_t other = __shfl_xor_sync(0xffffffffu, nmax, o); nmax = other > nmax ? other : nmax; }

    if (role == 1) {
        coop_produce<32>(&wk[0][0][0], lane, true, L, nfull, r, nblk, bits, nmax, one);
        return;
    }

    // ---------------- chain warp: 64 rounds per block on W+K from shared memory ------------------------
    const uint32_t minus_one = 0u - one;          // opaque like `one`: keeps the subtraction an IMAD
    (void)minus_one;
    uint32_t h[8];
    if (L.load_state) {
#pragma unroll
        for (int i = 0; i < 8; ++i) h[i] = j.state[8 * (uint64_t)L.sidx + i];
    } else {
        sha256_iv(h);
    }
    for (uint64_t b = 0; b < nmax; ++b) {
        const int st = (int)(b % kCoopStages);
        named_bar_sync(kFull0 + st, 64);
        if (b < nblk) {
            uint32_t s[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) s[i] = h[i];
#pragma unroll
            for (int g = 0; g < 16; ++g) {
                const uint4 v = wk[st][g][lane];
                const uint32_t wkq[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int t = 4 * g + q;
                    uint32_t& a = s[(0 - t) & 7]; uint32_t& bb = s[(1 - t) & 7]; uint32_t& c = s[(2 - t) & 7];
                    uint32_t& d = s[(3 - t) & 7]; uint32_t& e = s[(4 - t) & 7]; uint32_t& f = s[(5 - t) & 7];
                    uint32_t& gg = s[(6 - t) & 7]; uint32_t& hh = s[(7 - t) & 7];
                    if constexpr (VARIANT == 2) {
                        const uint32_t wkh = add_fma(wkq[q], hh, one);
                        const uint32_t x = add_fma(wkh, d, one);                 // no dependence on e: off the critical path
                        const uint32_t y = add_fma(x, ch(e, f, gg), one);
                        const uint32_t enew = add_fma(y, big_sigma1(e), one);
                        const uint32_t t1 = mad_lo(d, minus_one, enew);           // T1 = e' - d
                        const uint32_t z = add_fma(t1, maj(a, bb, c), one);
                        hh = add_fma(z, big_sigma0(a), one);
                        d = enew;
                    } else if constexpr (VARIANT == 0) {
                    // latency-bound warp: keep only one addition behind Sigma1 on the e-chain (one extra IMAD per round)
                    uint32_t y = add_fma(wkq[q], hh, one);
                    y = add_fma(y, ch(e, f, gg), one);
                    const uint32_t s1 = big_sigma1(e);
                    const uint32_t x = add_fma(d, y, one);
                    const uint32_t z = add_fma(y, maj(a, bb, c), one);
                    d = add_fma(x, s1, one);
                    const uint32_t z2 = add_fma(z, s1, one);
                    hh = add_fma(z2, big_sigma0(a), one);
                    } else {
                    uint32_t t1 = add_fma(wkq[q], hh, one);
                    t1 = add_fma(t1, ch(e, f, gg), one);
                    t1 = add_fma(t1, big_sigma1(e), one);
                    d = add_fma(d, t1, one);
                    const uint32_t t2 = add_fma(big_sigma0(a), maj(a, bb, c), one);
                    hh = add_fma(t1, t2, one);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) h[i] = add_fma(h[i], s[i], one);
        }
        if (b + kCoopStages < nmax) named_bar_arrive(kEmpty0 + st, 64);
    }
    if (!live) return;
    if (!fin) {
#pragma unroll
        for (int i = 0; i < 8; ++i) j.state[8 * (uint64_t)L.sidx + i] = h[i];
        return;
    }
    uint4 lo, hi;
    lo.x = bswap32(h[0]); lo.y = bswap32(h[1]); lo.z = bswap32(h[2]); lo.w = bswap32(h[3]);
    hi.x = bswap32(h[4]); hi.y = bswap32(h[5]); hi.z = bswap32(h[6]); hi.w = bswap32(h[7]);
    uint4* o = reinterpret_cast<uint4*>(j.out + 32 * (uint64_t)L.oidx);
    o[0] = lo; o[1] = hi;
}

// =====================================================================================================
// k_sha256_chains_pair: launches with very few chains (at most two CTAs per SM), where only the latency of ONE chain
// counts; bit for bit the same digests as k_sha256_chains_coop (the whole GPU test-suite runs through it).
// A chain is bound by the DEPENDENCY PATH of a round, e -> three rotates (issued 2 clk apart on the 16-lane pipe)
// -> xor3 -> add -> e' -- not by the 10 ALU-pipe instructions per round this kernel cuts to 8, nor by the 17 issue
// slots it cuts to 11.  What the split buys is ALU-pipe headroom, and that headroom is spent on the path: the final
// addition becomes one IADD3 on the pipe the rotates are on.
// Who gets here: a pushed file, the streamed tar.gz of the incremental hasher, the 32 shards of BASELINE config 3, the
// 1,000 blobs of config 5, every ring slot of a streamed tree digest.
// A warp instruction holds its sub-partition's 16-lane pipe for 2 clk whatever the number of active lanes, so the
// lanes of a warp are free to do different halves of the same round:
//   E lane (even)  holds e,f,g,h:  e' = Sigma1(e) + Ch(e,f,g) + h + W+K + d
//   A lane (odd)   holds a,b,c,d:  a' = Sigma0(a) + Maj(a,b,c) + (e' - d)
// Both are "xor of three rotates of v0, plus a three-input select, plus additions", so one instruction stream serves
// both with per-lane registers for what differs: the rotate amounts, Maj(a,b,c) = Ch(a, b|c, b&c) so that the select is
// the same LOP3 with operands prepared from OLD values (off the critical path), a +-1 multiplier and a zero column of
// W+K for the A lanes.  7 rotate/logic instructions per round instead of 10.  The lanes trade one value per round with
// ONE shfl.xor: E sends e', A sends a'.  The A lane runs two rounds behind the E lane, so what arrives is needed one
// iteration later (E needs d(t+1) = a(t-2), A needs e(t+1) - d(t) for its round t) and is added by the last instruction
// of that iteration.  A block is 66 iterations: 64 + the 2 of skew.  16 chains per CTA: chain warp + producer warp.
// Same MsgJob contract and the same results bit for bit as the other two kernels (tests/pair_pipeline_emulation.py is
// the dataflow in Python).
// =====================================================================================================
constexpr int kPairChains = 16;
constexpr int kPairStages = 4;                     // two pairs of blocks in flight
constexpr int kPairFull0 = 1, kPairEmpty0 = 3;     // named barriers per PAIR of blocks: full[2], empty[2]

template <int LUT>
__device__ __forceinline__ uint32_t lop3(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(LUT)); return d;
}

// Producer warp of the pair kernel.  Only 16 chains per CTA, so the warp's two halves work on two CONSECUTIVE blocks of
// the same 16 messages at once: lane L serves chain L & 15 and the blocks b = 2k + (L >> 4); one pass of the ~660
// instructions below (a single in-order warp needs well over a thousand clk for them) yields two blocks per chain.  Block b goes
// to stage b & 3; the chain warp is told per pair of blocks.
__device__ __forceinline__ void pair_produce(uint4 (*wk)[16][kPairChains + 1], const int lane, const Located& L, const uint64_t nfull,
                                             const uint32_t r, const uint64_t nblk, const uint64_t bits, const uint64_t nmax,
                                             const uint32_t one) {
    const uint8_t* ptr = L.ptr;
    const int chain = lane & (kPairChains - 1);
    const uint64_t half = (uint64_t)(lane >> 4);
    auto expand_store = [&](uint32_t (&w)[16], int st, bool publish) {
        constexpr K256Table K = k256_table();
#pragma unroll
        for (int g = 0; g < 16; ++g) {
            uint32_t o4[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int t = 4 * g + q;
                if (t >= 16) {
                    uint32_t x = add_fma(w[t & 15], small_sigma0(w[(t + 1) & 15]), one);
                    x = add_fma(x, w[(t + 9) & 15], one);
                    w[t & 15] = add_fma(x, small_sigma1(w[(t + 14) & 15]), one);
                }
                o4[q] = add_fma(w[t & 15], K.v[t], one);
            }
            if (publish) wk[st][g][chain] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
    };
    const bool warp_aligned = __all_sync(0xffffffffu, (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0);
    uint32_t w[16];
    uint64_t k = 0;                                   // pass k makes blocks 2k and 2k + 1
    if (warp_aligned) {
        // Hot loop: while every live chain has two more full blocks.  Lanes without a message shadow a live lane (same
        // address, same trip count, nothing published) so that they do not force the warp onto the slow path.
        const unsigned have = __ballot_sync(0xffffffffu, nblk > 0 && nfull > 0);
        const int src = have ? (__ffs(have) - 1) : 0;
        const uint64_t src_ptr = __shfl_sync(0xffffffffu, reinterpret_cast<uint64_t>(ptr), src);
        const uint64_t src_nfull = __shfl_sync(0xffffffffu, nfull, src);
        const bool shadow = (nblk == 0);
        const uint8_t* hot_ptr = shadow ? reinterpret_cast<const uint8_t*>(src_ptr) : ptr;
        const uint64_t hot_nfull = shadow ? src_nfull : nfull;
        uint64_t nfull_min = have ? hot_nfull : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const uint64_t other = __shfl_xor_sync(0xffffffffu, nfull_min, o); nfull_min = other < nfull_min ? other : nfull_min; }
        const uint64_t khot = nfull_min >> 1;         // passes in which both blocks are full for every lane
        if (khot > 0) {
            const uint4* p4 = reinterpret_cast<const uint4*>(hot_ptr) + 4 * half;
            uint4 v0 = ldg128(p4), v1 = ldg128(p4 + 1), v2 = ldg128(p4 + 2), v3 = ldg128(p4 + 3);
            for (; k < khot; ++k) {
                if (k >= 2) named_bar_sync(kPairEmpty0 + (int)(k & 1), 64);
                unpack_block(v0, v1, v2, v3, w);
                p4 += (2 * (k + 1) + half < hot_nfull) ? 8 : 0;     // my next block, if it is a full one (else re-read: L1 hit)
                v0 = ldg128(p4); v1 = ldg128(p4 + 1); v2 = ldg128(p4 + 2); v3 = ldg128(p4 + 3);
                expand_store(w, (int)((2 * k + half) & 3), !shadow);
                named_bar_arrive(kPairFull0 + (int)(k & 1), 64);
            }
        }
    }
    // Everything else: ragged tails of the batch, unaligned messages, padding and length blocks.
    for (; 2 * k < nmax; ++k) {
        if (k >= 2) named_bar_sync(kPairEmpty0 + (int)(k & 1), 64);
        const uint64_t b = 2 * k + half;
        if (b < nblk) {
            if (b < nfull) {
                load_block_unaligned(ptr + (b << 6), w);
            } else if (b == nfull) {
                const uint8_t* t = ptr + (nfull << 6);
#pragma unroll
                for (int kk = 0; kk < 16; ++kk) {
                    uint32_t word = 0;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t idx = 4 * kk + q;
                        if (idx < r) word |= (uint32_t)__ldg(t + idx) << (24 - 8 * q);
                        else if (idx == r) word |= 0x80u << (24 - 8 * q);
                    }
                    w[kk] = word;
                }
                if (r < 56) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
            } else {
#pragma unroll
                for (int kk = 0; kk < 14; ++kk) w[kk] = 0;
                w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
            }
            expand_store(w, (int)(b & 3), true);
        }
        named_bar_arrive(kPairFull0 + (int)(k & 1), 64);
    }
}

__global__ void __launch_bounds__(64) k_sha256_chains_pair(const MsgJob j) {
    // wk[stage][t/4][chain]; column kPairChains stays zero: the "W+K" of the A lanes
    __shared__ uint4 wk[kPairStages][16][kPairChains + 1];
    const int lane = threadIdx.x & 31;
    const int role = threadIdx.x >> 5;            // 0 = chain warp (lanes 2c, 2c+1 serve chain c), 1 = producer warp (lanes c, c+16)
    const int chain = role == 1 ? (lane & (kPairChains - 1)) : (lane >> 1);
    const uint64_t m = (uint64_t)blockIdx.x * kPairChains + chain;
    const uint32_t one = j.one;
    const Located L = locate(j, m);
    const uint64_t len = L.len;
    const bool live = L.live;
    const int fin = L.fin;
    const uint64_t nfull = len >> 6;
    const uint32_t r = (uint32_t)(len & 63u);
    const uint64_t nblk = live ? nfull + (fin ? (r >= 56 ? 2u : 1u) : 0u) : 0;
    const uint64_t bits = (L.prefix + len) << 3;
    uint64_t nmax = nblk;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const uint64_t other = __shfl_xor_sync(0xffffffffu, nmax, o); nmax = other > nmax ? other : nmax; }
    if (threadIdx.x < kPairStages * 16) wk[threadIdx.x >> 4][threadIdx.x & 15][kPairChains] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();

    if (role == 1) {
        pair_produce(wk, lane, L, nfull, r, nblk, bits, nmax, one);
        return;
    }

    // ---------------- chain warp ------------------------------------------------------------------------
    const bool isE = (lane & 1) == 0;
    const uint32_t r0 = isE ? 6u : 2u, r1 = isE ? 11u : 13u, r2 = isE ? 25u : 22u;   // Sigma1 / Sigma0
    const uint32_t coef = isE ? one : 0u - one;
    const uint32_t mA = isE ? 0u : 0xffffffffu;
    const int col = isE ? chain : kPairChains;
    uint32_t hs[4];                               // E lane: H4..H7, A lane: H0..H3
    if (L.load_state) {
#pragma unroll
        for (int i = 0; i < 4; ++i) hs[i] = j.state[8 * (uint64_t)L.sidx + (isE ? 4 : 0) + i];
    } else {
        uint32_t iv[8];
        sha256_iv(iv);
#pragma unroll
        for (int i = 0; i < 4; ++i) hs[i] = isE ? iv[4 + i] : iv[i];
    }
    for (uint64_t b = 0; b < nmax; ++b) {
        const int st = (int)(b & 3);
        const uint64_t pr2 = b >> 1;              // the pair of blocks this one belongs to
        if ((b & 1) == 0) named_bar_sync(kPairFull0 + (int)(pr2 & 1), 64);
        // Every lane runs every block of the longest chain (a finished pair computes on stale W+K and drops the result):
        // the warp stays converged, so the exchange is a bare SHFL with the full mask.
        {
            // window s[]: position p holds variable (p - i) mod 4 at iteration i.  E lane: (e,f,g,h).  A lane: (a,b,c,d),
            // which starts two rounds "before" round 0 as (H2, H3, -, -) and is fed H1, H0 in the two lead-in iterations,
            // so that the E lane receives d(1) = H2, d(2) = H1, d(3) = H0 through the ordinary exchange.
            uint32_t s[4];
            s[0] = isE ? hs[0] : hs[2]; s[1] = isE ? hs[1] : hs[3]; s[2] = hs[2]; s[3] = hs[3];
            uint4 v = wk[st][0][col];
            uint32_t recv_prev = __shfl_xor_sync(0xffffffffu, hs[3], 1);             // E receives H3 = d(0)
            uint32_t hwm_prev = mad_lo(hs[3], coef, v.x);                            // E: h(0) + W0+K0
            uint32_t e64[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int i = 0; i < 66; ++i) {
                uint32_t& v0 = s[(0 - i) & 3]; uint32_t& v1 = s[(1 - i) & 3]; uint32_t& v2 = s[(2 - i) & 3];
                uint32_t& v3 = s[(3 - i) & 3];
                const uint32_t recv = __shfl_xor_sync(0xffffffffu, v0, 1);           // consumed at the END of iteration i + 1
                const int t = i + 1;
                uint32_t wkx = 0u;
                if (t < 64) {
                    if ((t & 3) == 0) v = wk[st][t >> 2][col];
                    wkx = (t & 3) == 0 ? v.x : (t & 3) == 1 ? v.y : (t & 3) == 2 ? v.z : v.w;
                }
                const uint32_t x = xor3(__funnelshift_r(v0, v0, r0), __funnelshift_r(v0, v0, r1), __funnelshift_r(v0, v0, r2));
                const uint32_t p = lop3<0xF8>(v1, v2, mA);                           // E: f      A: b | c
                const uint32_t q = lop3<0xC4>(v1, v2, mA);                           // E: g      A: b & c
                const uint32_t c = ch(v0, p, q);                                     // E: Ch     A: Maj
                const uint32_t t1 = add_fma(c, hwm_prev, one);
                // The last addition is ONE three-input IADD3 on the ALU pipe, not two IMADs: this warp has ALU-pipe slots to spare
                // (8 of 12 per iteration), the hops Sigma -> add -> next rotate stay on one pipe, and the crossed value enters at
                // the very end, rather than ((C + hwm) + recv, then + X) as IMADs or hwm + recv pre-added (that IMAD is
                // scheduled early and waits for the shuffle).
                uint32_t nw = x + t1 + recv_prev;
                hwm_prev = mad_lo(v2, coef, wkx);                                    // E: h(t+1)+W+K(t+1)   A: -d(t+1)
                recv_prev = recv;
                if (i == 0) nw = isE ? nw : hs[1];
                if (i == 1) nw = isE ? nw : hs[0];
                v3 = nw;                                                             // v0 of the next iteration
                if (i == 63) { e64[0] = s[0]; e64[1] = s[1]; e64[2] = s[2]; e64[3] = s[3]; }   // (e,f,g,h) after round 63
            }
            // feed-forward (FIPS 180-4 section 6.2.2 step 4).  After iteration 65 the A lane's (a,b,c,d) sit in s[2],s[3],s[0],s[1].
#pragma unroll
            for (int k = 0; k < 4; ++k) hs[k] = b < nblk ? add_fma(hs[k], isE ? e64[k] : s[(k + 2) & 3], one) : hs[k];
        }
        // pair finished: its two stages may be refilled (only if the producer will come round to them again)
        if (((b & 1) == 1 || b + 1 == nmax) && 2 * (pr2 + 2) < nmax) named_bar_arrive(kPairEmpty0 + (int)(pr2 & 1), 64);
    }
    if (!live) return;
    if (!fin) {
#pragma unroll
        for (int i = 0; i < 4; ++i) j.state[8 * (uint64_t)L.sidx + (isE ? 4 : 0) + i] = hs[i];
        return;
    }
    uint4 o;
    o.x = bswap32(hs[0]); o.y = bswap32(hs[1]); o.z = bswap32(hs[2]); o.w = bswap32(hs[3]);
    reinterpret_cast<uint4*>(j.out + 32 * (uint64_t)L.oidx)[isE ? 1 : 0] = o;
}

// SHA-256 of a short message given as `nwords` big-endian 32-bit words (nwords a multiple of 8: concatenated
// digests), fetched through `word(i)`.  Tree nodes above the leaves: fanout * 8 words, 5 blocks for fanout 8.
template <typename F>
__device__ __forceinline__ void sha256_words(F word, const uint32_t nwords, uint32_t (&h)[8], const uint32_t one) {
    sha256_iv(h);
    const uint32_t nblk = (nwords * 4u + 9u + 63u) >> 6;
    uint32_t w[16];
    for (uint32_t b = 0; b < nblk; ++b) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const uint32_t wi = 16u * b + (uint32_t)k;
            w[k] = wi < nwords ? word(wi) : (wi == nwords ? 0x80000000u : 0u);
        }
        if (b + 1 == nblk) { w[14] = 0; w[15] = nwords * 32u; }
        sha256_compress(h, w, one);
    }
}

__device__ __forceinline__ void store_digest(uint8_t* out, const uint32_t (&h)[8]) {
    uint4 lo, hi;
    lo.x = bswap32(h[0]); lo.y = bswap32(h[1]); lo.z = bswap32(h[2]); lo.w = bswap32(h[3]);
    hi.x = bswap32(h[4]); hi.y = bswap32(h[5]); hi.z = bswap32(h[6]); hi.w = bswap32(h[7]);
    uint4* o = reinterpret_cast<uint4*>(out);
    o[0] = lo; o[1] = hi;
}

// =====================================================================================================
// k_tree_leaves: the leaf level of modelx.tree.v1 with the first tree levels fused in.
//
// Work unit = 64 consecutive leaves = one CTA pass: lane t hashes leaf 64u+t exactly like k_sha256_lanes, the 64
// digests meet in shared memory and the CTA reduces them through `fused` tree levels (fanout 8: 64 -> 8 -> 1, i.e.
// one digest per MiB leaves the kernel instead of 64), so levels 1..fused cost no launch, no DRAM round trip and no
// dependency tail behind the leaf launch.
//
// Scheduling.  Default (mode 1): one unit per CTA, the hardware block scheduler refills slots as CTAs finish.
// Mode 0 (MXD_TUNE_LEAF_SCHED=2, an A/B alternative, see launch_leaves_impl) tries to remove the
// drain at the end of a launch: a grid-scheduled launch ends with a drain in which the CTAs of an SM finish at
// scattered times and the last leaves run on a nearly empty machine.  Here the grid is exactly one CTA per resident slot (SMs x 12).  Every CTA looks up
// the SM it landed on (%smid) and takes a slot number there; SM s owns a contiguous share of the units, and its
// slots walk through that share in aligned rounds: with a units on the SM and 12 slots, q = ceil(a/12) units go to
// each of kmain = floor(a/q) >= 8 slots and the few left over to one more slot, which finishes early.  All kmain
// CTAs of an SM share its issue slots evenly, so they end together with >= 16 warps resident until the last block.
// Placement is not guaranteed by CUDA, so every unit is claimed with an atomic before it is hashed and a second,
// normally empty launch (mode 2) sweeps up any unit whose slot never showed up.  Results do not depend on who
// hashes what.  Small inputs (mode 1): one unit per CTA, grid = units.
// =====================================================================================================
constexpr uint32_t kMaxSmid = 1024;
constexpr uint32_t kSchedHeaderWords = 4 + 2 * kMaxSmid;

template <bool FUSED>
__global__ void __launch_bounds__(kThreads, 12) k_tree_leaves(const LeafJob j, const uint32_t n_units, const uint32_t nsm,
                                                              const uint32_t kper, const uint32_t mode, unsigned long long* dbg) {
    __shared__ uint32_t dig[FUSED ? 2 : 1][FUSED ? 64 : 1][8];
    __shared__ uint32_t s_info[4];
    unsigned long long t_begin = 0;
    if (dbg != nullptr && threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_begin));
    const uint32_t tid = threadIdx.x;
    const uint32_t one = j.one;
    uint32_t* const n_seen = j.sched;
    uint32_t* const sm_slots = j.sched + 4;
    uint32_t* const sm_dense = sm_slots + kMaxSmid;
    uint32_t* const claimed = sm_dense + kMaxSmid;

    uint32_t first = 0, stride = 1, count = 0;     // this CTA hashes units first + i*stride, i < count
    if (mode == 0) {
        if (tid == 0) {
            uint32_t smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            uint32_t slot = 0xffffffffu, dense = 0xffffffffu;
            if (smid < kMaxSmid) {
                slot = atomicAdd(&sm_slots[smid], 1u);
                if (slot == 0) {                    // first CTA on this SM: give the SM a dense index
                    dense = atomicAdd(n_seen, 1u);
                    atomicExch(&sm_dense[smid], dense + 1u);
                } else {                            // the slot-0 CTA is already running: its store arrives shortly
                    uint32_t v;
                    while ((v = atomicAdd(&sm_dense[smid], 0u)) == 0u) __nanosleep(20);
                    dense = v - 1u;
                }
            }
            s_info[0] = slot; s_info[1] = dense;
        }
        __syncthreads();
        const uint32_t slot = s_info[0], dense = s_info[1];
        if (dense < nsm) {
            uint32_t a = n_units / nsm;
            const uint32_t rem = n_units % nsm;
            const uint32_t u0 = dense * a + (dense < rem ? dense : rem);
            a += dense < rem ? 1u : 0u;
            const uint32_t q = (a + kper - 1) / kper;
            const uint32_t kmain = q ? a / q : 0u;
            if (slot < kmain) { first = u0 + slot; stride = kmain; count = q; }
            else if (slot == kmain) { first = u0 + kmain * q; stride = 1; count = a - kmain * q; }
        }
    } else {
        first = blockIdx.x; stride = gridDim.x;
        count = first < n_units ? (n_units - first + stride - 1) / stride : 0u;
    }

    uint32_t span = 1;
    for (uint32_t lv = 0; lv < j.fused; ++lv) span *= j.fanout;

    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t u = first + i * stride;
        if (mode != 1) {
            __syncthreads();                        // s_info[2] of the previous unit has been read by everyone
            if (tid == 0) s_info[2] = (mode == 2 && *reinterpret_cast<volatile uint32_t*>(&claimed[u]) != 0u)
                                          ? 1u : atomicCAS(&claimed[u], 0u, 1u);
            __syncthreads();
            if (s_info[2] != 0u) continue;
        }
        // ---- lane t: leaf 64u + t --------------------------------------------------------------------
        const uint64_t leaf_idx = (uint64_t)u * 64u + tid;
        const bool live = leaf_idx < j.n0;
        const uint64_t off = leaf_idx * j.leaf;
        const uint64_t len = (live && off < j.nbytes) ? ((j.nbytes - off < j.leaf) ? j.nbytes - off : j.leaf) : 0;
        const uint8_t* ptr = j.base + (live ? off : 0);
        const uint64_t nfull = len >> 6;
        const uint32_t r = (uint32_t)(len & 63u);
        const uint64_t nblk = live ? nfull + (r >= 56 ? 2u : 1u) : 0;
        uint32_t h[8];
        sha256_iv(h);
        absorb(ptr, nfull, r, nblk, len << 3, live, h, one);
        if constexpr (!FUSED) {
            if (live) store_digest(j.out + 32 * leaf_idx, h);
        } else {
        // ---- the tree levels that fit inside these 64 leaves, through shared memory -----------------------
#pragma unroll
        for (int k = 0; k < 8; ++k) dig[0][tid][k] = h[k];
        __syncthreads();
        const uint64_t left = j.n0 - (uint64_t)u * 64u;
        uint32_t cnt = left < 64u ? (uint32_t)left : 64u;
        uint32_t cur = 0;
        for (uint32_t lv = 0; lv < j.fused; ++lv) {
            const uint32_t nn = (cnt + j.fanout - 1) / j.fanout;
            if (tid < nn) {
                const uint32_t have = cnt - tid * j.fanout;
                const uint32_t nch = have < j.fanout ? have : j.fanout;
                const uint32_t* src = &dig[cur][tid * j.fanout][0];
                uint32_t g[8];
                sha256_words([&](uint32_t wi) { return src[wi]; }, nch * 8u, g, one);
#pragma unroll
                for (int k = 0; k < 8; ++k) dig[cur ^ 1][tid][k] = g[k];
            }
            __syncthreads();
            cur ^= 1; cnt = nn;
        }
        if (tid < cnt) {
            uint32_t g[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) g[k] = dig[cur][tid][k];
            store_digest(j.out + 32 * (((uint64_t)u * 64u) / span + tid), g);
        }
        __syncthreads();                            // dig[] is free for the next unit
        }
    }
    if (dbg != nullptr && threadIdx.x == 0) {       // developer aid (MXD_LEAF_DEBUG): where did this CTA run, when, how much
        unsigned long long t_end; uint32_t smid;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        unsigned long long* r = dbg + 4ull * blockIdx.x;
        r[0] = ((unsigned long long)smid << 32) | (mode == 0 ? s_info[0] : 0xffffu);
        r[1] = t_begin; r[2] = t_end; r[3] = count;
    }
}

// Everything above a short digest list in one CTA: levels while more than one node remains, then the 72-byte root
// message of modelx.tree.v1 (two blocks with padding).  scratch: two buffers of ceil(n/fanout)*32 bytes.
__global__ void __launch_bounds__(256) k_tree_top(const uint8_t* __restrict__ in, uint64_t n, const uint32_t fanout,
                                                  const uint64_t size, const uint64_t leaf, uint8_t* scratch,
                                                  uint8_t* __restrict__ root, const uint32_t one) {
    const uint64_t half = ((n + fanout - 1) / fanout) * 32;
    const uint8_t* cur = in;
    uint8_t* bufs[2] = {scratch, scratch + half};
    int which = 0;
    while (n > 1) {
        const uint64_t nn = (n + fanout - 1) / fanout;
        uint8_t* dst = bufs[which];
        for (uint64_t i = threadIdx.x; i < nn; i += blockDim.x) {
            const uint64_t have = n - i * fanout;
            const uint32_t nch = have < fanout ? (uint32_t)have : fanout;
            const uint32_t* src = reinterpret_cast<const uint32_t*>(cur + i * fanout * 32);
            uint32_t g[8];
            sha256_words([&](uint32_t wi) { return bswap32(src[wi]); }, nch * 8u, g, one);
            store_digest(dst + 32 * i, g);
        }
        __syncthreads();
        cur = dst; which ^= 1; n = nn;
    }
    if (threadIdx.x != 0) return;
    uint32_t m[18];   // the 72-byte root message as big-endian words
    m[0] = 0x6d6f6465u; m[1] = 0x6c782e74u; m[2] = 0x7265652eu; m[3] = 0x76310000u;   // "modelx.tree.v1\0\0"
    m[4] = bswap32((uint32_t)size); m[5] = bswap32((uint32_t)(size >> 32));              // LE64(size)
    m[6] = bswap32((uint32_t)leaf); m[7] = bswap32((uint32_t)(leaf >> 32));              // LE64(leaf)
    m[8] = bswap32(fanout); m[9] = 0;                                                     // LE32(fanout), LE32(0)
    const uint32_t* top = reinterpret_cast<const uint32_t*>(cur);
    for (int k = 0; k < 8; ++k) m[10 + k] = bswap32(top[k]);
    uint32_t h[8];
    sha256_iv(h);
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) w[k] = m[k];
    sha256_compress(h, w, one);
    w[0] = m[16]; w[1] = m[17]; w[2] = 0x80000000u;
#pragma unroll
    for (int k = 3; k < 15; ++k) w[k] = 0;
    w[15] = 72 * 8;
    sha256_compress(h, w, one);
    store_digest(root, h);
}

__global__ void k_compare(const uint8_t* __restrict__ got, const uint8_t* __restrict__ want, uint64_t n,
                          uint8_t* __restrict__ ok) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t diff = 0;
#pragma unroll
    for (int k = 0; k < 32; ++k) diff |= (uint32_t)(got[32 * i + k] ^ want[32 * i + k]);
    ok[i] = diff == 0;
}

__device__ __forceinline__ uint64_t splitmix64_at(uint64_t seed, uint64_t jdx) {
    uint64_t z = seed + (jdx + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void k_gen_fill(uint64_t* __restrict__ dst, uint64_t first_word, uint64_t nwords, uint64_t seed) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += stride)
        dst[i] = splitmix64_at(seed, first_word + i);
}

}  // namespace

// Occupancy: 24 warps per SM at 80 registers is the default; MXD_TUNE_MINB=8 (32 warps) and =4 (16 warps) keep the
// other builds selectable for A/B profiling.
static std::atomic<uint64_t> g_launches{0};
uint64_t kernel_launch_count() { return g_launches.load(); }

static int g_minb = [] { const char* e = getenv("MXD_TUNE_MINB"); const int v = e ? atoi(e) : 6; return (v == 8 || v == 4) ? v : 6; }();

// SM count of the current device (cached per device).
static int sm_count() {
    static int cache[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (cache[dev] == 0) {
        int sms = 0;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cache[dev] = sms > 0 ? sms : 1;
    }
    return cache[dev];
}

static long g_coop_max = [] { const char* e = getenv("MXD_TUNE_COOP"); return e ? atol(e) : 32768L; }();
// Very few chains (at most two 16-chain CTAs per SM, so that every warp has an SM sub-partition to itself): the
// two-lanes-per-chain kernel.  The threshold follows the SM count of the device (4,224 chains on a 132-SM H100).
// MXD_TUNE_PAIR=0 disables it, =N sets the threshold.
static long g_pair_max = [] { const char* e = getenv("MXD_TUNE_PAIR"); return e ? atol(e) : -1L; }();

cudaError_t launch_sha256(const MsgJob& job, cudaStream_t stream) {
    if (job.nmsg == 0) return cudaSuccess;
    const uint64_t blocks = (job.nmsg + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    // Few, long chains: two warps per 32 chains (see k_sha256_chains_coop); the lanes kernel wins once there are
    // tens of thousands of chains.  MXD_TUNE_COOP=0 disables, =N sets the threshold.
    const uint64_t pair_max = g_pair_max >= 0 ? (uint64_t)g_pair_max : 2ull * kPairChains * (uint64_t)sm_count();
    if (job.nmsg <= pair_max) {
        ++g_launches;
        k_sha256_chains_pair<<<(unsigned)((job.nmsg + kPairChains - 1) / kPairChains), 64, 0, stream>>>(job);
        return cudaGetLastError();
    }
    if (job.nmsg <= (uint64_t)g_coop_max) {
        const uint64_t cblocks = (job.nmsg + 31) / 32;
        ++g_launches;
        static const int chain = [] { const char* e = getenv("MXD_TUNE_CHAIN"); return e ? atoi(e) : 0; }();
        if (chain == 2)      k_sha256_chains_coop<2><<<(unsigned)cblocks, 64, 0, stream>>>(job);
        else if (chain == 1) k_sha256_chains_coop<1><<<(unsigned)cblocks, 64, 0, stream>>>(job);
        else                 k_sha256_chains_coop<0><<<(unsigned)cblocks, 64, 0, stream>>>(job);
        return cudaGetLastError();
    }
    static const int cta = [] { const char* e = getenv("MXD_TUNE_CTA"); return e ? atoi(e) : 64; }();
    if (cta == 32) {
        const uint64_t b32 = (job.nmsg + 31) / 32;
        if (b32 > 0x7fffffffull) return cudaErrorInvalidValue;
        ++g_launches;
        k_sha256_lanes<24, 32><<<(unsigned)b32, 32, 0, stream>>>(job);
        return cudaGetLastError();
    }
    if (g_minb == 8)      { ++g_launches; k_sha256_lanes<16><<<(unsigned)blocks, kThreads, 0, stream>>>(job); }
    else if (g_minb == 4) { ++g_launches; k_sha256_lanes<8><<<(unsigned)blocks, kThreads, 0, stream>>>(job); }
    else                  { ++g_launches; k_sha256_lanes<12><<<(unsigned)blocks, kThreads, 0, stream>>>(job); }
    return cudaGetLastError();
}

cudaError_t launch_compare(const uint8_t* got, const uint8_t* want, uint64_t n, uint8_t* ok, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    ++g_launches;
    k_compare<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(got, want, n, ok);
    return cudaGetLastError();
}

cudaError_t launch_gen_fill(void* dst, uint64_t offset, uint64_t n, uint64_t seed, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    if ((offset | n) & 7u || (reinterpret_cast<uintptr_t>(dst) & 7u)) return cudaErrorInvalidValue;
    const uint64_t nwords = n >> 3;
    uint64_t blocks = (nwords + 255) / 256;
    if (blocks > 64ull * sm_count()) blocks = 64ull * sm_count();
    ++g_launches;
    k_gen_fill<<<(unsigned)blocks, 256, 0, stream>>>(static_cast<uint64_t*>(dst), offset >> 3, nwords, seed);
    return cudaGetLastError();
}

// Resident CTAs per SM of the leaf kernel and the SM count of the current device (cached per device).
static void leaf_geometry(int* nsm, int* per_sm) {
    static int cache_occ[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (cache_occ[dev] == 0) {
        int occ = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_tree_leaves<false>, kThreads, 0);
        cache_occ[dev] = occ > 0 ? occ : 1;
    }
    *nsm = sm_count(); *per_sm = cache_occ[dev];
}

uint32_t leaf_fusable_levels(uint32_t fanout, uint32_t want) {
    // In-kernel tree levels are OFF by default: a level-1 pass has 8 live lanes and a level-2 pass 1, but each warp
    // instruction still holds the 16-lane ALU pipe for 2 clk, so the 10 extra block compressions per 64 leaves cost
    // several times the pipe time of the same nodes in wide launches.  MXD_TUNE_FUSE=1 enables them for A/B.
    static const bool on = [] { const char* e = getenv("MXD_TUNE_FUSE"); return e && atoi(e) > 0; }();
    if (!on) return 0;
    uint32_t lv = 0;
    uint64_t span = 1;
    while (lv < want && span * fanout <= 64 && 64 % (span * fanout) == 0) { span *= fanout; ++lv; }
    return lv;
}

bool leaf_kernel_selected() {
    static const bool on = [] {
        const char* f = getenv("MXD_TUNE_FUSE"); const char* s = getenv("MXD_TUNE_LEAF_SCHED");
        return (f && atoi(f) > 0) || (s && atoi(s) == 2);
    }();
    return on;
}

uint64_t leaf_sched_bytes(uint64_t n0) { return (kSchedHeaderWords + (n0 + 63) / 64) * sizeof(uint32_t); }

template <bool FUSED>
static cudaError_t launch_leaves_impl(const LeafJob& job, cudaStream_t stream) {
    const uint64_t units64 = (job.n0 + 63) / 64;
    if (units64 == 0 || units64 > 0x7fffffffull || job.sched == nullptr) return cudaErrorInvalidValue;
    const uint32_t n_units = (uint32_t)units64;
    int nsm = 1, per_sm = 1;
    leaf_geometry(&nsm, &per_sm);
    // 2: the persistent per-SM round schedule (mode 0 of k_tree_leaves); default: the hardware block scheduler.
    // Equal-work CTAs of one SM do not finish together -- the warp scheduler is greedy, not fair -- so static shares
    // end in a long low-occupancy tail.  Dynamic refill avoids it.
    static const int tune = [] { const char* e = getenv("MXD_TUNE_LEAF_SCHED"); return e ? atoi(e) : 1; }();
    static const int kper_env = [] { const char* e = getenv("MXD_TUNE_LEAF_KPER"); return e ? atoi(e) : 0; }();  // CTAs per SM (A/B)
    if (kper_env > 0 && kper_env < per_sm) per_sm = kper_env;
    const uint32_t resident = (uint32_t)nsm * (uint32_t)per_sm;
    if (tune != 2 || n_units < 2 * resident || (uint32_t)nsm > kMaxSmid) {
        // small input (or A/B): plain grid, one unit per CTA (mode 1 with grid == units)
        ++g_launches;
        k_tree_leaves<FUSED><<<n_units, kThreads, 0, stream>>>(job, n_units, (uint32_t)nsm, (uint32_t)per_sm, 1u, nullptr);
        return cudaGetLastError();
    }
    static const char* dbg_path = getenv("MXD_LEAF_DEBUG");
    unsigned long long* dbg = nullptr;
    if (dbg_path) cudaMalloc(&dbg, 32ull * resident);
    cudaError_t e = cudaMemsetAsync(job.sched, 0, leaf_sched_bytes(job.n0), stream);
    if (e != cudaSuccess) return e;
    ++g_launches;
    k_tree_leaves<FUSED><<<resident, kThreads, 0, stream>>>(job, n_units, (uint32_t)nsm, (uint32_t)per_sm, 0u, dbg);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // sweep: hashes whatever unit is still unclaimed (none when every SM received its per_sm CTAs)
    ++g_launches;
    k_tree_leaves<FUSED><<<(unsigned)nsm, kThreads, 0, stream>>>(job, n_units, (uint32_t)nsm, (uint32_t)per_sm, 2u, nullptr);
    e = cudaGetLastError();
    if (dbg) {      // developer aid: per-SM placement and timing of the persistent launch, appended to $MXD_LEAF_DEBUG
        cudaStreamSynchronize(stream);
        std::vector<unsigned long long> h(4ull * resident);
        cudaMemcpy(h.data(), dbg, 32ull * resident, cudaMemcpyDeviceToHost);
        cudaFree(dbg);
        if (FILE* f = fopen(dbg_path, "a")) {
            unsigned long long t0 = ~0ull, t1 = 0;
            for (uint32_t i = 0; i < resident; ++i) { if (h[4 * i + 1] && h[4 * i + 1] < t0) t0 = h[4 * i + 1]; if (h[4 * i + 2] > t1) t1 = h[4 * i + 2]; }
            fprintf(f, "launch units=%u nsm=%d per_sm=%d span_us=%.1f\n", n_units, nsm, per_sm, (t1 - t0) / 1e3);
            for (uint32_t i = 0; i < resident; ++i)
                fprintf(f, "cta %u smid %llu slot %llu start_us %.1f end_us %.1f units %llu\n", i, h[4 * i] >> 32, h[4 * i] & 0xffffffffull,
                        (h[4 * i + 1] - t0) / 1e3, (h[4 * i + 2] - t0) / 1e3, h[4 * i + 3]);
            fclose(f);
        }
    }
    return e;
}

cudaError_t launch_tree_leaves(const LeafJob& job, cudaStream_t stream) {
    return job.fused ? launch_leaves_impl<true>(job, stream) : launch_leaves_impl<false>(job, stream);
}

// scratch layout: two buffers of ceil(n/fanout)*32 bytes for the wide levels, then 16 KiB for k_tree_top's own
// ping-pong (at most 512 digests enter it, so at most 256 * 32 bytes per buffer).
constexpr uint64_t kTopNarrow = 512;
uint64_t tree_top_scratch_bytes(uint64_t n, uint32_t fanout) { return 2 * (((n + fanout - 1) / fanout) * 32) + 2 * (kTopNarrow / 2) * 32; }

cudaError_t launch_tree_top(const uint8_t* digests, uint64_t n, uint32_t fanout, uint64_t size, uint64_t leaf,
                            uint8_t* scratch, uint8_t* root, cudaStream_t stream) {
    if (n == 0 || fanout < 2) return cudaErrorInvalidValue;
    // wide levels first (thousands of nodes want the whole machine), the narrow rest and the root in one CTA
    const uint64_t half = ((n + fanout - 1) / fanout) * 32;
    const uint8_t* cur = digests;
    int which = 0;
    while (n > kTopNarrow) {
        MsgJob j{};
        j.base = cur; j.nbytes = n * 32; j.seg = 32ull * fanout; j.nmsg = (n + fanout - 1) / fanout;
        j.out = scratch + (which ? half : 0); j.finalize = 1; j.one = 1;
        cudaError_t e = launch_sha256(j, stream);
        if (e != cudaSuccess) return e;
        cur = j.out; which ^= 1; n = j.nmsg;
    }
    ++g_launches;
    k_tree_top<<<1, 256, 0, stream>>>(cur, n, fanout, size, leaf, scratch + 2 * half, root, 1u);
    return cudaGetLastError();
}

int sha256_kernel_regs() {
    cudaFuncAttributes a;
    if (cudaFuncGetAttributes(&a, k_sha256_lanes<12>) != cudaSuccess) return -1;
    return a.numRegs;
}

}  // namespace mxd
