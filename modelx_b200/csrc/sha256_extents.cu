// Tree leaves of a blob that is scattered over device buffers (mxd_dev_tree_digest_extents): a safetensors checkpoint
// in HBM is a header plus a few hundred tensor allocations, and its tree digest is that of their concatenation.
//
// One lane per leaf, 64-thread CTAs, 12 CTAs per SM (the same 80-register budget as k_sha256_lanes).  Leaf i is the
// logical range [i*leaf, min((i+1)*leaf, size)) of the concatenation; lane i of a launch hashes leaf first + i, so a
// streaming caller (mxd_tree_load_file) can hash one ring slot's leaves at a time against the whole table.  A lane
// binary-searches the extent table for the extent holding its first byte and then walks forward through the table.
//
// Fast loop: while every lane of a group has its next blocks wholly inside one extent and all of them share the same
// address class a = addr & 15, the group runs a straight-line loop specialised on a (the warp-minimum number of blocks
// left before any member's extent boundary), prefetching the next block while compressing the current one:
//   a == 0        4 x LDG.128 per block, exactly the loop of k_sha256_lanes;
//   a != 0        the 5 aligned 16-byte vectors that cover the block; the fifth is the first of the next block, so it is
//                 carried over and a block costs 4 x LDG.128 as well.  Word k of the block is one PRMT of two adjacent
//                 loaded words: the byte offset a & 3 and the byte swap are the same selector, so this class issues
//                 the same 16 PRMTs per block as the aligned one and no other instruction on the ALU pipe.
// Consecutive leaves inside one tensor always qualify (leaf sizes are multiples of 64), so only warps that meet a tensor
// boundary leave the fast loop.  Lanes with another class wait and run next; a block that straddles two extents, the
// padded tail block and the length block go through a byte-at-a-time path that is correct for any layout, including a
// leaf made of hundreds of tiny extents.
#include "kernels.h"
#include "sha256_device.cuh"

namespace mxd {

namespace {

constexpr int kThreads = 64;
constexpr unsigned kAll = 0xffffffffu;

// A lane's read position: the device address of its next byte and how many bytes of that extent are left from there.
struct Cursor {
    const uint8_t* p;
    uint64_t left;
    uint64_t e;
};

__device__ __forceinline__ void enter(Cursor& c, const DevExtent* ext, uint64_t e) {
    c.e = e;
    c.p = static_cast<const uint8_t*>(ext[e].ptr);
    c.left = ext[e].len;
}

// The extent holding byte `pos` (< size): the last one whose start is <= pos.  Extents are non-empty and in order.
__device__ __forceinline__ Cursor locate_byte(const DevExtent* ext, uint64_t m, uint64_t pos) {
    uint64_t lo = 0, hi = m - 1;
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) >> 1;
        if (ext[mid].start <= pos) lo = mid; else hi = mid - 1;
    }
    Cursor c;
    enter(c, ext, lo);
    const uint64_t skip = pos - ext[lo].start;
    c.p += skip; c.left -= skip;
    return c;
}

// k >= 1 full blocks at p, 16-byte aligned.
__device__ __forceinline__ void blocks_aligned(const uint8_t* p, const uint64_t k, uint32_t (&h)[8], const uint32_t one) {
    const uint4* p4 = reinterpret_cast<const uint4*>(p);
    uint4 v0 = ldg128(p4), v1 = ldg128(p4 + 1), v2 = ldg128(p4 + 2), v3 = ldg128(p4 + 3);
    for (uint64_t b = 0; b < k; ++b) {
        uint32_t w[16];
        unpack_block(v0, v1, v2, v3, w);
        p4 += (b + 1 < k) ? 4 : 0;   // last iteration re-reads its own block (L1 hit) instead of branching
        v0 = ldg128(p4); v1 = ldg128(p4 + 1); v2 = ldg128(p4 + 2); v3 = ldg128(p4 + 3);
        sha256_compress(h, w, one);
    }
}

// k >= 1 full blocks at p, where p & 15 = 4 W + s is not 0; sel is the PRMT selector of byte offset s.  The block is
// bytes [4W + s, 4W + s + 64) of the 80 loaded from the aligned address below p; all five vectors hold block bytes, so
// no load leaves the 16-byte granules of the extent.
template <int W>
__device__ __forceinline__ void blocks_shifted(const uint8_t* p, const uint64_t k, const uint32_t sel, uint32_t (&h)[8],
                                               const uint32_t one) {
    const uint4* q = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(p) & ~static_cast<uintptr_t>(15));
    uint4 v0 = ldg128(q), v1 = ldg128(q + 1), v2 = ldg128(q + 2), v3 = ldg128(q + 3), v4 = ldg128(q + 4);
    for (uint64_t b = 0; b < k; ++b) {
        const uint32_t x[20] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y,
                                v2.z, v2.w, v3.x, v3.y, v3.z, v3.w, v4.x, v4.y, v4.z, v4.w};
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = __byte_perm(x[W + i], x[W + i + 1], sel);
        q += (b + 1 < k) ? 4 : 0;
        v0 = v4;                     // the next block's first vector is this block's last
        v1 = ldg128(q + 1); v2 = ldg128(q + 2); v3 = ldg128(q + 3); v4 = ldg128(q + 4);
        sha256_compress(h, w, one);
    }
}

// The lane's next block, read one byte at a time through its cursor: nb message bytes, then the 0x80 marker when `pad`,
// zeros after.  Crosses into the following extent(s) as needed; nb bytes must exist.
__device__ __forceinline__ void gather_block(Cursor& c, const DevExtent* ext, const uint32_t nb, const bool pad,
                                             uint32_t (&w)[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t idx = 4 * k + q;
            if (idx < nb) {
                if (c.left == 0) enter(c, ext, c.e + 1);
                word |= (uint32_t)__ldg(c.p) << (24 - 8 * q);
                ++c.p; --c.left;
            } else if (idx == nb && pad) {
                word |= 0x80u << (24 - 8 * q);
            }
        }
        w[k] = word;
    }
}

__global__ void __launch_bounds__(kThreads, 12) k_tree_leaves_extents(const ExtentLeafJob j) {
    const uint64_t lane = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
    const uint32_t one = j.one;
    const bool live = lane < j.n0;
    const uint64_t lo = (j.first + lane) * j.leaf;
    const uint64_t len = (live && lo < j.size) ? ((j.size - lo < j.leaf) ? j.size - lo : j.leaf) : 0;
    const uint64_t nfull = len >> 6;
    const uint32_t r = (uint32_t)(len & 63u);
    const uint64_t nblk = live ? nfull + (r >= 56 ? 2u : 1u) : 0;
    const uint64_t bits = len << 3;
    Cursor c{nullptr, 0, 0};
    if (len) c = locate_byte(j.ext, j.m, lo);
    uint32_t h[8];
    sha256_iv(h);
    uint64_t b = 0;
    while (__any_sync(kAll, b < nblk)) {
        if (b < nfull && c.left == 0) enter(c, j.ext, c.e + 1);
        const bool inside = b < nfull && c.left >= 64;
        const unsigned fast = __ballot_sync(kAll, inside);
        // A block that straddles two extents holds up the whole warp for one byte-wise step; anything else that is not
        // wholly inside an extent (tail and length blocks) waits until no lane has a fast block left.
        if (fast != 0u && !__any_sync(kAll, b < nfull && !inside)) {
            const uint32_t mine = (uint32_t)reinterpret_cast<uintptr_t>(c.p) & 15u;
            const uint32_t a = __shfl_sync(kAll, mine, __ffs(fast) - 1);
            const bool run = inside && mine == a;
            uint64_t k = run ? ((nfull - b < (c.left >> 6)) ? nfull - b : (c.left >> 6)) : ~0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const uint64_t other = __shfl_xor_sync(kAll, k, o); k = other < k ? other : k; }
            if (run) {
                if (a == 0) {
                    blocks_aligned(c.p, k, h, one);
                } else {
                    const uint32_t s = a & 3u;
                    const uint32_t sel = ((s + 3u)) | ((s + 2u) << 4) | ((s + 1u) << 8) | (s << 12);
                    switch (a >> 2) {
                        case 0: blocks_shifted<0>(c.p, k, sel, h, one); break;
                        case 1: blocks_shifted<1>(c.p, k, sel, h, one); break;
                        case 2: blocks_shifted<2>(c.p, k, sel, h, one); break;
                        default: blocks_shifted<3>(c.p, k, sel, h, one); break;
                    }
                }
                c.p += k << 6; c.left -= k << 6; b += k;
            }
            continue;
        }
        if (b < nblk) {
            uint32_t w[16];
            const bool tail = b >= nfull;
            gather_block(c, j.ext, tail ? (b == nfull ? r : 0u) : 64u, b == nfull, w);
            if (b > nfull || (tail && r < 56)) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
            sha256_compress(h, w, one);
            ++b;
        }
    }
    if (live) store_digest(j.out + 32 * lane, h);
}

}  // namespace

cudaError_t launch_tree_leaves_extents(const ExtentLeafJob& job, cudaStream_t stream) {
    if (job.n0 == 0 || (job.size != 0 && (job.m == 0 || job.ext == nullptr)) || job.out == nullptr) return cudaErrorInvalidValue;
    const uint64_t blocks = (job.n0 + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    count_kernel_launch();
    k_tree_leaves_extents<<<(unsigned)blocks, kThreads, 0, stream>>>(job);
    return cudaGetLastError();
}

}  // namespace mxd
