/*
 * modelx_digest.h -- C ABI of libmodelxdigest.so, the H100-native digest-and-chunk engine that
 * replaces the CPU hot path of kubegems/modelx push/pull.
 *
 * The reference (Go, CGO_ENABLED=0) has no FFI; the seams this ABI replaces are plain Go calls.
 * Each entry point below cites the reference call site (file:line under the modelx tree) whose
 * work it takes over.  INTEGRATION.md shows the cgo binding a maintainer would add.
 *
 * Conventions
 *   - Every function is thread-safe and re-entrant (the reference calls the path from up to 3
 *     goroutines per Push/Pull, pkg/client/push.go:27, progress/mbar.go:47-51).
 *   - Return value: MXD_OK (0) or a negative mxd_status.  The caller owns every buffer; the
 *     library keeps no pointer after a call returns (except the mxd_dev_* enqueue calls, which
 *     are asynchronous on the given CUDA stream, as documented there).
 *   - Digests are raw 32-byte SHA-256 values; mxd_digest_string() renders the reference's
 *     "sha256:<64 hex>" form (go-digest v1.0.0 Digest.String()).
 *   - There is NO CPU fallback: without a usable CUDA device mxd_open fails with
 *     MXD_ERR_NO_DEVICE and nothing else can be called.
 *   - Plain C types only: pointers, sizes, integers.  Device pointers are raw CUDA device
 *     addresses (e.g. torch.Tensor.data_ptr()), streams are cudaStream_t passed as void*.
 */
#ifndef MODELX_DIGEST_H
#define MODELX_DIGEST_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MXD_ABI_VERSION 2

typedef enum mxd_status {
    MXD_OK = 0,
    MXD_ERR_INVALID = -1,      /* bad argument (reference: would be a Go panic or DIGEST_INVALID, pkg/errors/errors.go:69) */
    MXD_ERR_NO_DEVICE = -2,    /* no CUDA device / driver: the engine refuses to run on the CPU */
    MXD_ERR_CUDA = -3,         /* a CUDA call failed; mxd_last_error() has the text (maps to INTERNAL, errors.go:65) */
    MXD_ERR_IO = -4,           /* open/read failed; errno preserved (reference returns the os error) */
    MXD_ERR_NOMEM = -5,
    MXD_ERR_CANCELED = -6,     /* the call's operation was canceled (reference: ctx cancel closes the fd, push.go:156-159) */
    MXD_ERR_DIV_ZERO = -7      /* calcParts with 0 parts: the reference panics (extension_s3.go:100) */
} mxd_status;

typedef struct mxd_ctx mxd_ctx;
typedef struct mxd_hasher mxd_hasher;
typedef struct { const void* ptr; uint64_t len; } mxd_span;   /* host or device memory */
typedef struct { int64_t offset, length; } mxd_part;          /* PartRange{offset,length}, extension_s3.go:91-97 */

typedef struct {
    uint64_t kernel_launches;   /* kernels this library has launched in this process (every launch counts one) */
    uint64_t bytes_hashed;      /* message bytes submitted to the SHA-256 kernel */
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t src_bytes_read;    /* bytes read from files / copied out of host buffers into the pinned ring (read-once accounting) */
    uint64_t open_files;        /* files the digest service holds open right now (bounded, see MXD_MAX_OPEN_FILES) */
    uint64_t reserved[2];
} mxd_stats;

/* Environment knobs (read once, at mxd_open / first launch):
 *   MXD_RING_BYTES      pinned + device ring size per device in bytes (overrides the ring_bytes argument)
 *   MXD_STAGE_THREADS   threads per device that fill ring slots from files / pageable memory (default min(16, cpus/devices))
 *   MXD_STAGE_PIECE     bytes each filler thread reads at a time (default 1 MiB)
 *   MXD_STAGE_MMAP=1    stage files out of a read-only mapping with streaming stores instead of pread (SIGBUS-guarded);
 *                       faster only when few CPUs are available (measured: 2 CPUs +17 %, 16 CPUs -32 %), off by default
 *   MXD_NO_NUMA_BIND    set to disable binding pinned allocations and filler threads to the device's local CPUs
 *   MXD_MAX_OPEN_FILES  files the whole-message digest service may hold open at once (default RLIMIT_NOFILE/2 - 32, capped at 4096)
 *   MXD_TUNE_COOP       largest launch (in messages) that uses the two-warp cooperative kernel (default 32768, 0 = never)
 *   MXD_TUNE_PAIR       largest launch (in messages) that uses the two-lanes-per-chain kernel (default 4736 = two CTAs per SM, 0 = never)
 *   MXD_TUNE_MINB=8     select the 63-register build of the lanes kernel (A/B profiling only)
 *   MXD_TUNE_CHAIN=1|2  other ways of writing the round in the two-warp chain kernel; MXD_TUNE_CTA=32: one-warp CTAs in the lanes
 *                       kernel (both measured: no gain; A/B only)
 *   MXD_TUNE_LEAF_SCHED=2       leaf kernel as a persistent grid with a static per-SM round schedule (measured slower; A/B only)
 *   MXD_TUNE_FUSE=1             first tree levels inside the leaf kernel (measured slower: 8-lane warps hold the ALU pipe; A/B only) */

/* ---- lifecycle ------------------------------------------------------------------------- */
/* devices/ndev: CUDA ordinals to drive from this process (ndev == 0: all visible devices).
 * ring_bytes: pinned host ring + device ring per device for streaming host data (0 = default). */
int  mxd_open(mxd_ctx** out, const int* devices, int ndev, uint64_t ring_bytes);
void mxd_close(mxd_ctx* ctx);
int  mxd_device_count(const mxd_ctx* ctx);
/* ---- operations: per-call cancellation ----------------------------------------------------
 * The reference cancels ONE digest through that call's own context (push.go:150-159: ctx.Done closes the fd) and
 * the first failing blob cancels its siblings through their shared context (progress/mbar.go:108-115).  An
 * operation handle is that context: mxd_op_begin returns a handle that can be passed wherever an mxd_ctx* is
 * accepted (it shares the devices, rings and digest service of its parent); mxd_cancel(op) makes every call made
 * through THAT handle -- running or future -- return MXD_ERR_CANCELED and touches nobody else.  One operation per
 * call gives push.go:150-159; one operation shared by the blobs of a Push gives mbar.go:108-115.
 * mxd_cancel(root handle) aborts every call that is in flight on the context at that moment (process shutdown);
 * it is not sticky: calls started afterwards run normally. */
int  mxd_op_begin(mxd_ctx* parent, mxd_ctx** op);
void mxd_op_end(mxd_ctx* op);               /* after the last call through it has returned */
void mxd_cancel(mxd_ctx* handle);
void mxd_reset_cancel(mxd_ctx* op);         /* un-cancel an operation handle (no effect on a root handle) */
int  mxd_is_canceled(const mxd_ctx* op);
int  mxd_get_stats(const mxd_ctx* ctx, mxd_stats* out);
/* Live kernel timing for benchmarks: while enabled, every leaf-level SHA-256 launch (the launch
 * that reads blob bytes) is bracketed by CUDA events on its own stream.  mxd_prof_read waits for
 * them and returns the accumulated device time, launch count and message bytes, then clears. */
int  mxd_prof_enable(mxd_ctx* ctx, int on);
int  mxd_prof_read(mxd_ctx* ctx, double* kernel_ms, uint64_t* launches, uint64_t* bytes);
/* Slot timeline of the streaming ring (overlap evidence without a system profiler): while enabled, every ring slot
 * of the tree path records host fill time and CUDA events around its H2D copy and its kernel; mxd_trace_dump writes
 * them as CSV (times in ms since the first record's copy start, per device) and clears the record. */
int  mxd_trace_enable(mxd_ctx* ctx, int on);
int  mxd_trace_dump(mxd_ctx* ctx, const char* csv_path);
const char* mxd_strerror(int status);
const char* mxd_last_error(void);           /* thread-local detail of the last failure on this thread */
int  mxd_abi_version(void);

/* ---- whole-message digests: the reference's semantics ------------------------------------
 * digest.FromBytes / digest.FromReader: one SHA-256 over the whole byte string.
 * One message is one serial chain, so a single call runs on a single GPU lane; throughput
 * comes from batching many messages (mxd_sha256_batch / mxd_sha256_files). */
int mxd_sha256(mxd_ctx*, const void* data, uint64_t n, uint8_t out[32]);                 /* digest.Canonical.FromBytes, push.go:25 */
int mxd_sha256_batch(mxd_ctx*, const mxd_span* spans, uint64_t n, uint8_t* out /*n*32*/);  /* n x FromBytes, host or device spans */
int mxd_sha256_file(mxd_ctx*, const char* path, uint8_t out[32], uint64_t* size);        /* Client.digest, push.go:149-161; pull.go:116 */
int mxd_sha256_files(mxd_ctx*, const char* const* paths, uint64_t n, uint8_t* out /*n*32*/,
                     uint64_t* sizes /*n, may be NULL*/);                                /* Push/PullBlobs fan-out, push.go:36-52, pull.go:41-50 */
/* The general form behind the calls above: one job per file, each with its own status, so one unreadable or
 * canceled file does not fail its siblings.  A job may ask for the SHA-256 of several byte ranges of its file --
 * e.g. {0,size} and every calcParts range (extension_s3.go:99-112) -- and may tee every byte of the file to a sink
 * (a part uploader / store writer): the file is then read from disk ONCE, where the reference reads it once to hash
 * (push.go:160) and once more to upload (extension_s3.go:71-82).  All jobs of a call, and all calls in flight from
 * other threads, advance together as lanes of the same GPU rounds.  Sink contract: called with disjoint pieces (<= 4 MiB)
 * that together cover the file exactly once, possibly concurrently from several threads and in any order; the data pointer
 * is only valid during the call; a sink must not call back into this library (it runs inside a service round); a non-zero
 * return fails that file with MXD_ERR_IO. */
typedef int (*mxd_sink_fn)(void* user, uint64_t offset, const void* data, uint64_t nbytes);
typedef struct {
    const char* path;
    const mxd_part* ranges; uint64_t nranges;   /* nranges == 0: one digest of the whole file */
    uint8_t* out;                               /* max(nranges, 1) * 32 bytes */
    mxd_sink_fn sink; void* sink_user;          /* may be NULL */
    uint64_t size;                              /* out: file size */
    int status;                                 /* out: MXD_OK or this file's error */
} mxd_file_job;
int mxd_sha256_file_jobs(mxd_ctx*, mxd_file_job* jobs, uint64_t n);   /* returns MXD_OK or the first failing job's status */
int mxd_sha256_file_ranges(mxd_ctx*, const char* path, const mxd_part* ranges, uint64_t n, uint8_t* out /*n*32*/,
                           uint64_t* size, mxd_sink_fn sink, void* sink_user);
/* Routing advice for callers that still own a CPU SHA-256 (the Go client's crypto/sha256): 1 when hashing this many
 * blobs together on the GPU is expected to beat the reference's 3 goroutines on SHA-NI cores, else 0.  A single
 * whole-file digest is one serial chain and never pays off; see INTEGRATION.md section 3 for the measured table. */
int mxd_batch_pays_off(uint64_t n_blobs, uint64_t total_bytes, uint64_t max_blob_bytes);
/* pull.go:115-123: "do I already have this blob?"  ok[i] = 1 iff SHA-256(span i) == want[i]. */
int mxd_verify_batch(mxd_ctx*, const mxd_span* spans, const uint8_t* want /*n*32*/, uint64_t n, uint8_t* ok /*n*/);
int mxd_verify_files(mxd_ctx*, const char* const* paths, const uint8_t* want /*n*32*/, uint64_t n, uint8_t* ok /*n*/);

/* ---- incremental hasher: hash.Hash shape for TGZ's io.MultiWriter (helper.go:46-49) --------
 * write never fails for lack of data; sum does not disturb the state (Go: Sum appends a copy). */
int  mxd_hasher_new(mxd_ctx*, mxd_hasher** out);
int  mxd_hasher_write(mxd_hasher*, const void* data, uint64_t n);
int  mxd_hasher_sum(mxd_hasher*, uint8_t out[32]);
int  mxd_hasher_reset(mxd_hasher*);
uint64_t mxd_hasher_size(const mxd_hasher*);        /* hash.Hash.Size(): 32 */
uint64_t mxd_hasher_block_size(const mxd_hasher*);  /* hash.Hash.BlockSize(): 64 */
uint64_t mxd_hasher_written(const mxd_hasher*);     /* bytes written so far */
void mxd_hasher_free(mxd_hasher*);

/* ---- chunked tree digest (new; what lets one blob use every lane and every GPU) -----------
 * "modelx.tree.v1" with parameters (leaf, fanout, chunk = leaf * fanout^k, k >= 1):
 *   level 0:  leaf i = SHA-256 of bytes [i*leaf, (i+1)*leaf)   (n0 = max(1, ceil(size/leaf)) leaves)
 *   level j+1: node i = SHA-256 of the concatenated level-j digests [i*fanout, (i+1)*fanout)
 *   levels are built at least up to level k -- whose nodes each cover `chunk` bytes: these are the
 *   CHUNK DIGESTS, the list a manifest carries -- and further while a level has more than one node;
 *   top = the single digest of the last level;
 *   root = SHA-256("modelx.tree.v1\0\0" || LE64(size) || LE64(leaf) || LE32(fanout) || LE32(0) || top).
 * Every node is a plain SHA-256 of well-defined bytes (bit-exact vs crypto/sha256 on those bytes).
 * The root is NOT the reference's whole-file digest (push.go:160); see DESIGN.md section 3.
 * A NULL params pointer means the defaults: chunk 8 MiB, leaf 16 KiB, fanout 8. */
typedef struct {
    uint64_t chunk;     /* bytes per chunk digest; leaf * fanout^k */
    uint64_t leaf;      /* bytes hashed by one GPU lane; multiple of 64 */
    uint32_t fanout;    /* digests per upper-level node; >= 2 */
    uint32_t reserved;  /* 0 */
} mxd_tree_params;

int mxd_tree_shape(uint64_t size, const mxd_tree_params* tp, uint64_t* counts, int max_levels,
                   int* chunk_level); /* returns #levels */
int mxd_tree_digest(mxd_ctx*, const void* data /*host or device*/, uint64_t size, const mxd_tree_params* tp,
                    uint8_t* chunk_digests /*nchunks*32, may be NULL*/, uint64_t* nchunks, uint8_t root[32]);
int mxd_tree_digest_file(mxd_ctx*, const char* path, const mxd_tree_params* tp,
                         uint8_t* chunk_digests, uint64_t cap_chunks, uint64_t* nchunks, uint64_t* size, uint8_t root[32]);
/* Read-once form (SURVEY 8f.1): the same digest, and every byte that streams through the pinned ring is also
 * handed to `sink` (e.g. a part uploader or a store writer), so the file is read from disk once instead of once to
 * hash and once to upload (push.go:160 then extension_s3.go:71-82).  The sink is called with disjoint pieces
 * (<= 4 MiB) that together cover [0, size), possibly concurrently from several threads and in any order; the data
 * pointer is only valid during the call.  A non-zero return aborts the digest with MXD_ERR_IO. */
int mxd_tree_digest_file_tee(mxd_ctx*, const char* path, const mxd_tree_params* tp, uint8_t* chunk_digests,
                             uint64_t cap_chunks, uint64_t* nchunks, uint64_t* size, uint8_t root[32],
                             mxd_sink_fn sink, void* user);
/* Tree roots of MANY files in one pipelined pass (e.g. the pull-side check of a manifest whose blobs are tree keyed): the
 * files stream through the ring back to back, so the copy engine and the SMs do not drain between files.  roots: n*32;
 * sizes and status (per file, MXD_OK or that file's I/O error) may be NULL.  Returns MXD_OK or the first failing status. */
int mxd_tree_digest_files(mxd_ctx*, const char* const* paths, uint64_t n, const mxd_tree_params* tp, uint8_t* roots,
                          uint64_t* sizes, int* status);
/* Sharded form (one process per GPU): chunk digests of a piece that starts on a chunk boundary... */
int mxd_tree_chunks(mxd_ctx*, const void* piece /*host or device*/, uint64_t nbytes, const mxd_tree_params* tp,
                    uint8_t* chunk_digests /*max(1, ceil(nbytes/chunk))*32*/);
/* The same for a piece of a FILE: bytes [offset, offset+nbytes) of `path`, offset a multiple of the chunk size.  What a
 * rank of a sharded push calls for its chunk range; streams through the pinned ring like mxd_tree_digest_file. */
int mxd_tree_chunks_file(mxd_ctx*, const char* path, uint64_t offset, uint64_t nbytes, const mxd_tree_params* tp,
                         uint8_t* chunk_digests /*max(1, ceil(nbytes/chunk))*32*/);
/* ...and the levels above the gathered chunk list (the only step after the all-gather). */
int mxd_tree_finish(mxd_ctx*, const uint8_t* chunk_digests, uint64_t nchunks, uint64_t size,
                    const mxd_tree_params* tp, uint8_t root[32]);

/* ---- multipart split: integer-only, bit-exact with the reference ------------------------- */
int     mxd_calc_parts(int64_t total, int64_t partscount, mxd_part* out /*partscount*/);   /* calcParts, extension_s3.go:99-112 */
int64_t mxd_server_part_count(int64_t size, int force_multipart);                         /* store_s3.go:198-203,273-279 */

/* SHA-256 of each part [offset, offset+length) of one file, all parts advanced together as one GPU batch:
 * the ranges S3Extension.Upload sends (extension_s3.go:52-89 over calcParts), e.g. for per-part
 * x-amz-checksum-sha256.  New (the reference never hashes a part); each digest is the plain SHA-256 of that
 * byte range.  Ranges may overlap or leave gaps; a range past EOF is MXD_ERR_IO. */
int mxd_sha256_file_parts(mxd_ctx*, const char* path, const mxd_part* parts, uint64_t n, uint8_t* out /*n*32*/);

/* ---- digest strings (go-digest v1.0.0; registry.go:218-227 BlobDigestFun accepts only this form) */
void mxd_digest_string(const uint8_t d[32], char out[72]);      /* "sha256:" + 64 lower hex + NUL */
int  mxd_digest_parse(const char* s, uint8_t out[32]);          /* MXD_ERR_INVALID unless exactly that form */

/* ---- pinned host memory for callers that want zero-copy H2D -------------------------------- */
int  mxd_host_alloc(mxd_ctx*, void** out, uint64_t nbytes);
void mxd_host_free(mxd_ctx*, void* p);
int  mxd_host_register(mxd_ctx*, void* p, uint64_t nbytes);
int  mxd_host_unregister(mxd_ctx*, void* p);

/* ---- device-resident, asynchronous forms ---------------------------------------------------
 * Inputs and outputs are device pointers on device `dev` (index into the context's device list);
 * work is enqueued on `stream` (a cudaStream_t; NULL = the legacy default stream) and the call
 * returns without synchronising.  Used by bench.py (kernel-only timing) and by callers that
 * already hold blobs in HBM.
 * Alignment: message bytes (d_data, d_piece, span pointers) may start at any address.  Digest
 * outputs (d_out, d_chunk_digests, d_root) and the chunk-digest input of mxd_dev_tree_finish must
 * be 16-byte aligned, d_spans 8-byte aligned, and mxd_dev_gen_fill's d_dst, offset and n multiples
 * of 8.  A data pointer may be NULL only when its length is 0.  A call that breaks one of these
 * rules returns MXD_ERR_INVALID and enqueues nothing. */
int mxd_dev_sha256_segments(mxd_ctx*, int dev, const void* d_data, uint64_t nbytes, uint64_t seg,
                            void* d_out /*ceil(nbytes/seg)*32*/, void* stream);
int mxd_dev_sha256_batch(mxd_ctx*, int dev, const mxd_span* d_spans /*device array*/, uint64_t n, void* d_out, void* stream);
int mxd_dev_tree_chunks(mxd_ctx*, int dev, const void* d_piece, uint64_t nbytes, const mxd_tree_params* tp,
                        void* d_chunk_digests, void* stream);
int mxd_dev_tree_finish(mxd_ctx*, int dev, const void* d_chunk_digests, uint64_t nchunks, uint64_t size,
                        const mxd_tree_params* tp, void* d_root /*32*/, void* stream);
int mxd_dev_tree_digest(mxd_ctx*, int dev, const void* d_data, uint64_t size, const mxd_tree_params* tp,
                        void* d_chunk_digests /*may be NULL*/, void* d_root /*32*/, void* stream);
int mxd_dev_compare(mxd_ctx*, int dev, const void* d_got, const void* d_want, uint64_t n, void* d_ok /*n bytes*/, void* stream);
/* deterministic synthetic blob (benchmarks/tests): LE64 word j = splitmix64(seed, j); offset, n multiples of 8 */
int mxd_dev_gen_fill(mxd_ctx*, int dev, void* d_dst, uint64_t offset, uint64_t n, uint64_t seed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MODELX_DIGEST_H */
