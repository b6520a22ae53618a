// Internal (non-ABI) interface between the CUDA kernels and the C-ABI layer.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace mxd {

// Per-message descriptor of one round of the digest service (mxd_lockstep.cu): where this round's
// bytes of the message sit on the device, how much of the message earlier rounds absorbed, which
// persistent chain-state slot it owns and what to do at the end of the round.
struct LaneDesc {
    const void* ptr;   // this round's bytes (device memory, any alignment)
    uint64_t len;      // multiple of 64 unless kFinalize is set
    uint64_t prefix;   // bytes absorbed by earlier rounds (multiple of 64)
    uint32_t lane;     // index of the chain state (8 words) in MsgJob::state
    uint32_t oidx;     // index of the 32-byte digest in MsgJob::out (only read when kFinalize)
    uint32_t ctl;      // kFinalize | kSkip | kFresh
    uint32_t pad;
};
enum : uint32_t { kFinalize = 1u, kSkip = 2u, kFresh = 4u };   // kFresh: start from the FIPS 180-4 IV, ignore stored state

// One launch hashes `nmsg` independent messages, one SHA-256 chain per lane.
struct MsgJob {
    // --- where message m lives (first non-null of descs / base / spans wins) ------------------
    // uniform segments of one buffer (tree levels, chunk ranges): ptr = base + m*seg,
    // len = min(seg, nbytes - m*seg); nbytes == 0 means one empty message.
    const uint8_t* base;
    uint64_t nbytes;
    uint64_t seg;
    // arbitrary spans (batches of blobs): spans[m] = {ptr, len}, device memory.
    const void* spans;
    // digest-service rounds: descs[m], device memory (chained mode with per-message control).
    const LaneDesc* descs;
    uint64_t nmsg;
    // --- results ---------------------------------------------------------------------------
    uint8_t* out;            // 32 bytes per finalized message
    // --- chained mode (streaming a message through several launches) -------------------------
    uint32_t* state;         // nullable; 8 words per message/lane, read at start, written when not finalizing
    uint64_t prefix_all;     // bytes already absorbed (base/spans mode)
    int finalize;            // base/spans mode: 1 pad and emit digest; 0 len must be a multiple of 64
    uint32_t one;            // must be 1: opaque multiplier that steers additions to the FMA pipe
};

struct DevSpan { const void* ptr; uint64_t len; };

// The leaf level of a tree digest with the first tree levels fused into the same kernel: every CTA hashes 64
// consecutive leaves (one per lane) and then, through shared memory, the tree nodes above them for as many levels
// as fit inside 64 leaves (`fused` levels, fanout^fused <= 64); only the top fused level is written to memory.
// Persistent: the grid is one CTA per resident slot, each SM works through its own contiguous share of the
// 64-leaf units in aligned rounds (see k_tree_leaves).
struct LeafJob {
    const uint8_t* base;     // blob bytes
    uint64_t nbytes;
    uint64_t leaf;           // bytes per leaf, multiple of 64
    uint64_t n0;             // number of leaves = max(1, ceil(nbytes / leaf))
    uint32_t fanout;         // >= 2
    uint32_t fused;          // tree levels computed inside the CTA (0: the kernel writes the leaf digests)
    uint8_t* out;            // digests of level `fused`: ceil(n0 / fanout^fused) * 32 bytes
    uint32_t* sched;         // device scratch: kSchedWords words, zeroed by the launcher before every launch
    uint32_t one;
};

cudaError_t launch_sha256(const MsgJob& job, cudaStream_t stream);
// Tree leaves (+ fused levels).  `sched` is device scratch of leaf_sched_bytes() bytes owned by the caller's device
// state; a launch may not overlap another launch using the same scratch.
cudaError_t launch_tree_leaves(const LeafJob& job, cudaStream_t stream);
uint64_t leaf_sched_bytes(uint64_t n0);
// true when an A/B knob (MXD_TUNE_FUSE=1, MXD_TUNE_LEAF_SCHED=2) selects k_tree_leaves; by default tree leaves go through
// launch_sha256 like every other level (both experiments measured slower, see sha256_kernels.cu)
bool leaf_kernel_selected();
// How many tree levels launch_tree_leaves will fuse for this fanout when asked for at most `want` levels.
uint32_t leaf_fusable_levels(uint32_t fanout, uint32_t want);
// One piece of a blob that is scattered over device buffers: `len` (> 0) bytes at `ptr` (any alignment), which are bytes
// [start, start + len) of the concatenation.
struct DevExtent { const void* ptr; uint64_t len; uint64_t start; };

// The leaf level of a tree digest over a concatenation of extents, or a window of it: leaf i = SHA-256 of bytes
// [i*leaf, min((i+1)*leaf, size)) of the concatenation (one empty leaf when size == 0).  A launch hashes leaves
// [first, first + n0) and writes leaf first + i to out + 32 i; only those leaves' bytes are read.
struct ExtentLeafJob {
    const DevExtent* ext;    // device table of m extents in concatenation order (may be NULL when m == 0)
    uint64_t m;
    uint64_t size;           // sum of the extent lengths
    uint64_t leaf;           // bytes per leaf, multiple of 64
    uint64_t n0;             // leaves in this launch; first + n0 <= max(1, ceil(size / leaf))
    uint8_t* out;            // n0 * 32 bytes, 16-byte aligned
    uint32_t one;
    uint64_t first;          // index of the first leaf (0: the whole leaf level when n0 covers it)
};
cudaError_t launch_tree_leaves_extents(const ExtentLeafJob& job, cudaStream_t stream);

// All levels above a digest list (n >= 1 digests of 32 bytes, groups of `fanout`) and the root message, one launch:
// root = SHA256("modelx.tree.v1\0\0" || LE64(size) || LE64(leaf) || LE32(fanout) || LE32(0) || top[32]).
// scratch: device memory of tree_top_scratch_bytes(n, fanout) bytes.
cudaError_t launch_tree_top(const uint8_t* digests, uint64_t n, uint32_t fanout, uint64_t size, uint64_t leaf,
                            uint8_t* scratch, uint8_t* root, cudaStream_t stream);
uint64_t tree_top_scratch_bytes(uint64_t n, uint32_t fanout);
// ok[i] = (memcmp(got + 32 i, want + 32 i, 32) == 0)
cudaError_t launch_compare(const uint8_t* got, const uint8_t* want, uint64_t n, uint8_t* ok, cudaStream_t stream);
// bytes [offset, offset+n) of the splitmix64 counter stream (offset and n multiples of 8, dst 8-byte aligned)
cudaError_t launch_gen_fill(void* dst, uint64_t offset, uint64_t n, uint64_t seed, cudaStream_t stream);
int sha256_kernel_regs();
// kernels this library has launched in this process (every <<<>>> of the library counts one)
uint64_t kernel_launch_count();
void count_kernel_launch();

}  // namespace mxd
