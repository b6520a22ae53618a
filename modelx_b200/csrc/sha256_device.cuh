// SHA-256 block function for sm_90a, written for the SM's integer issue structure.
//
// Each of the four SM sub-partitions has a 16-lane ALU pipe (SHF/LOP3/IADD3/PRMT) and a separate
// FMA pipe that also executes IMAD, so additions written as IMADs issue beside the logic ops
// (tools/ubench/pipes.cu measures the rates).  FIPS 180-4 SHA-256 needs 672 shifts/rotates +
// 352 three-input logic ops + 16 byte swaps per 64-byte block that can only run on the ALU
// pipe (1040 ops), plus ~600 two-input additions that can run on either.  ptxas by default
// emits most additions as IADD3 (ALU pipe), making the ALU pipe carry ~1280 ops/block.  Here
// every addition is written as  a*1+b  with the 1 held in a register the compiler cannot see
// through, so it becomes an IMAD on the otherwise idle FMA pipe and the ALU pipe only carries
// the 1040 ops that have no alternative.  Ceiling: 4 SMSP * 32 lanes * 64 B / (1040 * 2 clk)
// = 3.94 B/clk/SM.
//
// Algorithm: FIPS 180-4 sections 4.1.2 (functions), 4.2.2 (constants), 6.2.2 (compression).
// Reference call sites this serves: pkg/client/push.go:160, pull.go:116, helper.go:46
// (digest.FromReader / Digester -> go-digest v1.0.0 -> crypto/sha256).
#pragma once
#include <cstdint>

namespace mxd {

// Round constants (FIPS 180-4 section 4.2.2) as a constexpr table so fully unrolled rounds take them as
// instruction immediates (no constant-bank or shared-memory read on the critical path).
struct K256Table { uint32_t v[64]; };
__host__ __device__ constexpr K256Table k256_table() {
    return K256Table{{
        0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
        0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
        0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
        0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
        0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
        0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
        0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
        0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u}};
}

__device__ __forceinline__ void sha256_iv(uint32_t (&h)[8]) {
    h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
    h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
}

// ---- primitive ops, each pinned to the pipe we want it on ------------------------------------
// ALU pipe
__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }      // SHF.R.W
__device__ __forceinline__ uint32_t xor3(uint32_t a, uint32_t b, uint32_t c) {                        // LOP3 0x96
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t ch(uint32_t e, uint32_t f, uint32_t g) {                           // LOP3 0xCA
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0xCA;" : "=r"(d) : "r"(e), "r"(f), "r"(g)); return d;
}
__device__ __forceinline__ uint32_t maj(uint32_t a, uint32_t b, uint32_t c) {                          // LOP3 0xE8
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }         // PRMT

// FMA pipe: a + b computed as a*one + b where `one` is an opaque register holding 1.
// MXD_ADD_ON_ALU=1 switches back to plain adds (ptxas then picks IADD3), kept for A/B profiling.
// MXD_ADD_IMM=1 writes the 1 as an immediate (mad.lo a,1,b): ptxas then sees through it and turns two thirds of the
// additions back into IADD3 (SASS of the leaf kernel: 494 IADD3 / 238 IMAD.IADD), which is why the 1 is opaque.
#ifndef MXD_ADD_ON_ALU
#define MXD_ADD_ON_ALU 0
#endif
__device__ __forceinline__ uint32_t add_fma(uint32_t a, uint32_t b, uint32_t one) {
#if MXD_ADD_ON_ALU
    (void)one; return a + b;
#elif defined(MXD_ADD_IMM) && MXD_ADD_IMM
    (void)one; uint32_t d; asm("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d;   // A/B: IMAD.IADD (immediate 1)
#else
    uint32_t d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(b)); return d;
#endif
}

__device__ __forceinline__ uint32_t big_sigma0(uint32_t x) { return xor3(rotr(x, 2), rotr(x, 13), rotr(x, 22)); }
__device__ __forceinline__ uint32_t big_sigma1(uint32_t x) { return xor3(rotr(x, 6), rotr(x, 11), rotr(x, 25)); }
__device__ __forceinline__ uint32_t small_sigma0(uint32_t x) { return xor3(rotr(x, 7), rotr(x, 18), x >> 3); }
__device__ __forceinline__ uint32_t small_sigma1(uint32_t x) { return xor3(rotr(x, 17), rotr(x, 19), x >> 10); }

// The 64 rounds on s[8] in place (no feed-forward).  w[16] holds the block as big-endian words and
// is clobbered (rolling 16-word schedule kept in registers).  `one` must hold 1 (see add_fma).
__device__ __forceinline__ void sha256_rounds(uint32_t (&s)[8], uint32_t (&w)[16], uint32_t one) {
    constexpr K256Table K = k256_table();
#pragma unroll
    for (int t = 0; t < 64; ++t) {
        if (t >= 16) {
            // W[t] = sigma1(W[t-2]) + W[t-7] + sigma0(W[t-15]) + W[t-16]
            uint32_t x = add_fma(w[t & 15], small_sigma0(w[(t + 1) & 15]), one);
            x = add_fma(x, w[(t + 9) & 15], one);
            w[t & 15] = add_fma(x, small_sigma1(w[(t + 14) & 15]), one);
        }
        // register renaming instead of moving a..h: position p holds variable (p - t) mod 8
        uint32_t& a = s[(0 - t) & 7]; uint32_t& b = s[(1 - t) & 7]; uint32_t& c = s[(2 - t) & 7];
        uint32_t& d = s[(3 - t) & 7]; uint32_t& e = s[(4 - t) & 7]; uint32_t& f = s[(5 - t) & 7];
        uint32_t& g = s[(6 - t) & 7]; uint32_t& hh = s[(7 - t) & 7];
        uint32_t t1 = add_fma(w[t & 15], K.v[t], one);        // off the critical path
        t1 = add_fma(t1, hh, one);
        t1 = add_fma(t1, ch(e, f, g), one);
        t1 = add_fma(t1, big_sigma1(e), one);
        d = add_fma(d, t1, one);                              // becomes e of the next round
        uint32_t t2 = add_fma(big_sigma0(a), maj(a, b, c), one);
        hh = add_fma(t1, t2, one);                            // becomes a of the next round
    }
}

// One 512-bit block: rounds + feed-forward (FIPS 180-4 section 6.2.2 step 4).
__device__ __forceinline__ void sha256_compress(uint32_t (&h)[8], uint32_t (&w)[16], uint32_t one) {
    uint32_t s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = h[i];
    sha256_rounds(s, w, one);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = add_fma(h[i], s[i], one);
}

// ---- block loads and digest stores shared by the kernels -----------------------------------------
__device__ __forceinline__ uint4 ldg128(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

__device__ __forceinline__ void unpack_block(const uint4& v0, const uint4& v1, const uint4& v2, const uint4& v3,
                                             uint32_t (&w)[16]) {
    w[0] = bswap32(v0.x);  w[1] = bswap32(v0.y);  w[2] = bswap32(v0.z);  w[3] = bswap32(v0.w);
    w[4] = bswap32(v1.x);  w[5] = bswap32(v1.y);  w[6] = bswap32(v1.z);  w[7] = bswap32(v1.w);
    w[8] = bswap32(v2.x);  w[9] = bswap32(v2.y);  w[10] = bswap32(v2.z); w[11] = bswap32(v2.w);
    w[12] = bswap32(v3.x); w[13] = bswap32(v3.y); w[14] = bswap32(v3.z); w[15] = bswap32(v3.w);
}

__device__ __forceinline__ void store_digest(uint8_t* out, const uint32_t (&h)[8]) {
    uint4 lo, hi;
    lo.x = bswap32(h[0]); lo.y = bswap32(h[1]); lo.z = bswap32(h[2]); lo.w = bswap32(h[3]);
    hi.x = bswap32(h[4]); hi.y = bswap32(h[5]); hi.z = bswap32(h[6]); hi.w = bswap32(h[7]);
    uint4* o = reinterpret_cast<uint4*>(out);
    o[0] = lo; o[1] = hi;
}

}  // namespace mxd
