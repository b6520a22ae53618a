// C ABI of libmodelxdigest.so (include/modelx_digest.h): handles and operations, the pinned-host ring that
// streams host/file data to the GPUs, tree assembly, device-resident forms and the integer split helpers.
// Host side of the hot path of kubegems/modelx push/pull; each entry point cites the reference call site it
// replaces in the header.  There is deliberately no CPU hashing in this library: if CUDA is unavailable every
// digest call fails.
#include "mxd_core.h"

#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <fcntl.h>
#include <fstream>
#include <memory>
#include <sys/resource.h>
#include <sys/stat.h>
#include <unistd.h>

namespace mxdi {

namespace {
thread_local std::string g_last_error;
}
int fail(int status, const std::string& msg) { g_last_error = msg; return status; }
const std::string& last_error() { return g_last_error; }

const uint32_t kIVHost[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};

namespace {

// MXD_DEBUG_TIMING=1: print host-side phase timings of the streaming calls to stderr (developer aid)
const bool g_dbg_timing = getenv("MXD_DEBUG_TIMING") != nullptr;
struct PhaseTimer {
    const char* what; timespec t0;
    explicit PhaseTimer(const char* w) : what(w) { if (g_dbg_timing) clock_gettime(CLOCK_MONOTONIC, &t0); }
    ~PhaseTimer() {
        if (!g_dbg_timing) return;
        timespec t1; clock_gettime(CLOCK_MONOTONIC, &t1);
        fprintf(stderr, "[mxd] %-28s %9.3f ms\n", what, (t1.tv_sec - t0.tv_sec) * 1e3 + (t1.tv_nsec - t0.tv_nsec) * 1e-6);
    }
};
double now_ms() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; }

constexpr uint64_t kDefaultRingBytes = 256ull << 20;

}  // namespace

// ---- NUMA locality ------------------------------------------------------------------------------------
// On an 8-GPU HGX board four GPUs hang off each CPU socket.  Pinned buffers that end up on the other
// socket cross the inter-socket link on every H2D copy, so pinned allocations and the slot-filler threads are bound to the CPUs that are local to the
// device (sysfs local_cpulist of its PCI function).  Best effort: any failure leaves affinity untouched.
bool device_local_cpus(int ordinal, cpu_set_t* set) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, ordinal) != cudaSuccess) { cudaGetLastError(); return false; }
    for (char* p = bus; *p; ++p) *p = (char)tolower(*p);
    std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist");
    std::string list;
    if (!f || !std::getline(f, list) || list.empty()) return false;
    CPU_ZERO(set);
    int count = 0;
    size_t i = 0;
    while (i < list.size()) {
        char* end = nullptr;
        long a = strtol(list.c_str() + i, &end, 10), b = a;
        if (end == list.c_str() + i) break;
        i = (size_t)(end - list.c_str());
        if (i < list.size() && list[i] == '-') { b = strtol(list.c_str() + i + 1, &end, 10); i = (size_t)(end - list.c_str()); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, set); ++count; }
        if (i < list.size() && list[i] == ',') ++i;
    }
    return count > 0;
}

LocalCpuScope::LocalCpuScope(int ordinal) {
    cpu_set_t want;
    if (getenv("MXD_NO_NUMA_BIND") || !device_local_cpus(ordinal, &want)) return;
    if (sched_getaffinity(0, sizeof old, &old) != 0) return;
    cpu_set_t both; CPU_AND(&both, &old, &want);            // stay inside whatever the container allows
    if (CPU_COUNT(&both) == 0) return;
    active = sched_setaffinity(0, sizeof both, &both) == 0;
}
LocalCpuScope::~LocalCpuScope() { if (active) sched_setaffinity(0, sizeof old, &old); }

// ---- StagePool -------------------------------------------------------------------------------------------
StagePool::StagePool(int nthreads) {
    for (int i = 0; i < nthreads; ++i) workers_.emplace_back([this] { run(); });
}
StagePool::~StagePool() {
    { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
}
void StagePool::parallel_for(int n, const std::function<void(int)>& fn) {
    if (n <= 0) return;
    if (n == 1 || workers_.empty()) { for (int i = 0; i < n; ++i) fn(i); return; }
    Batch b; b.fn = &fn; b.n = n; b.next = 0; b.done = 0;
    { std::lock_guard<std::mutex> lk(mu_); queue_.push_back(&b); }
    cv_.notify_all();
    for (;;) {  // the caller works too
        int i = b.next.fetch_add(1);
        if (i >= n) break;
        fn(i);
        b.done.fetch_add(1);
    }
    std::unique_lock<std::mutex> lk(mu_);
    for (auto it = queue_.begin(); it != queue_.end(); ++it) if (*it == &b) { queue_.erase(it); break; }
    done_cv_.wait(lk, [&] { return b.done.load() >= n && b.active == 0; });
}
void StagePool::run() {
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
        cv_.wait(lk, [&] { return stop_ || !queue_.empty(); });
        if (stop_) return;
        Batch* b = queue_.front();
        if (b->next.load() >= b->n) { queue_.erase(queue_.begin()); continue; }
        b->active++;
        lk.unlock();
        for (;;) {
            int i = b->next.fetch_add(1);
            if (i >= b->n) break;
            (*b->fn)(i);
            b->done.fetch_add(1);
        }
        lk.lock();
        b->active--;
        done_cv_.notify_all();
    }
}

MemKind classify(const void* p, int* device_ordinal) {
    cudaPointerAttributes a{};
    if (p == nullptr || cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return MemKind::Pageable; }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
        if (device_ordinal) *device_ordinal = a.device;
        return MemKind::Device;
    }
    if (a.type == cudaMemoryTypeHost) return MemKind::Pinned;
    return MemKind::Pageable;
}

int dev_index_of(const Core* c, int ordinal) {
    for (size_t i = 0; i < c->devs.size(); ++i)
        if (c->devs[i]->ordinal == ordinal) return (int)i;
    return -1;
}

DevState* pick_device(Core* c) { return c->devs[c->rr++ % c->devs.size()]; }

// hand [off, off+n) (already staged at `data`) to the tee in <= 4 MiB pieces, in parallel on the pool
int sink_pieces(const Source& s, uint64_t off, uint64_t n, const uint8_t* data, StagePool* pool) {
    if (!s.sink || n == 0) return MXD_OK;
    constexpr uint64_t kPiece = 4ull << 20;
    const int pieces = (int)((n + kPiece - 1) / kPiece);
    std::atomic<int> bad{0};
    auto put = [&](int i) {
        const uint64_t p0 = (uint64_t)i * kPiece, pn = std::min(kPiece, n - p0);
        if (s.sink(s.sink_user, s.sink_base + off + p0, data + p0, pn) != 0) bad.store(1);
    };
    if (pool && pieces > 1) pool->parallel_for(pieces, put); else for (int i = 0; i < pieces; ++i) put(i);
    return bad.load() ? fail(MXD_ERR_IO, "sink refused data") : MXD_OK;
}

int source_stage(Core* c, const Source& s, uint64_t off, uint64_t n, uint8_t* dst, const uint8_t** from, StagePool* pool) {
    if (s.fd < 0 && s.pinned) { *from = s.mem + off; return MXD_OK; }
    *from = dst;
    static const uint64_t kPiece = [] { const char* e = getenv("MXD_STAGE_PIECE"); uint64_t v = e ? strtoull(e, nullptr, 10) : 0; return v >= 4096 ? v : (1ull << 20); }();
    const int pieces = (int)((n + kPiece - 1) / kPiece);
    std::atomic<int> err{0};
    auto fill = [&](int i) {
        const uint64_t p0 = (uint64_t)i * kPiece, pn = std::min(kPiece, n - p0);
        if (s.map) {          // mapped file: streaming-store copy out of the page cache, under the SIGBUS guard
            if (stage_copy_mapped(dst + p0, s.map + off + p0, pn) != 0) err.store(-1);
        } else if (s.fd >= 0) {
            uint64_t got = 0;
            while (got < pn) {
                ssize_t r = pread(s.fd, dst + p0 + got, pn - got, (off_t)(s.base + off + p0 + got));
                if (r < 0) { if (errno == EINTR) continue; err.store(errno ? errno : EIO); return; }
                if (r == 0) { err.store(-1); return; }
                got += (uint64_t)r;
            }
        } else {
            stage_copy(dst + p0, s.mem + off + p0, pn);
        }
    };
    if (pool && pieces > 1) pool->parallel_for(pieces, fill);
    else for (int i = 0; i < pieces; ++i) fill(i);
    const int e = err.load();
    if (e == -1) return fail(MXD_ERR_IO, "read: file shrank while hashing");
    if (e) return fail(MXD_ERR_IO, std::string("pread: ") + strerror(e));
    c->src_read += n;
    return MXD_OK;
}

namespace {

// Resolved tree parameters: chunk = leaf * fanout^klevel.
struct Tree {
    uint64_t chunk = 8ull << 20, leaf = 16ull << 10, fanout = 8;
    int klevel = 3;
};

bool tree_resolve(const mxd_tree_params* tp, Tree* t) {
    if (tp) { t->chunk = tp->chunk; t->leaf = tp->leaf; t->fanout = tp->fanout; }
    if (t->leaf < 64 || (t->leaf % 64) != 0 || t->fanout < 2 || t->chunk < t->leaf) return false;
    if (tp && tp->reserved != 0) return false;
    uint64_t span = t->leaf;
    int k = 0;
    while (span < t->chunk) {
        if (span > t->chunk / t->fanout) return false;   // overflow / not a power
        span *= t->fanout; ++k;
    }
    if (span != t->chunk || k < 1) return false;
    t->klevel = k;
    return true;
}

uint64_t ipow(uint64_t b, uint32_t e) { uint64_t r = 1; while (e--) r *= b; return r; }

// ---- live timing of leaf launches --------------------------------------------------------------------------
struct ProfScope {
    Core* c; Core::ProfRec rec{}; bool on = false; cudaStream_t st;
    ProfScope(Core* core, uint64_t nbytes, cudaStream_t stream, bool enabled = true) : c(core), st(stream) {
        if (!enabled || !c->prof_on.load()) return;
        { std::lock_guard<std::mutex> lk(c->prof_mu); if (c->prof.size() >= (1u << 16)) return; }   // bounded
        cudaGetDevice(&rec.ordinal);
        if (cudaEventCreate(&rec.a) != cudaSuccess) return;
        if (cudaEventCreate(&rec.b) != cudaSuccess) { cudaEventDestroy(rec.a); return; }
        rec.bytes = nbytes;
        cudaEventRecord(rec.a, st);
        on = true;
    }
    ~ProfScope() {
        if (!on) return;
        cudaEventRecord(rec.b, st);
        std::lock_guard<std::mutex> lk(c->prof_mu);
        c->prof.push_back(rec);
    }
};

// ---- kernel enqueue helpers ------------------------------------------------------------------
// uniform segments of device memory -> one digest each (plain SHA-256 per segment)
int enqueue_segments(Core* c, const uint8_t* d_data, uint64_t nbytes, uint64_t seg, uint8_t* d_out, cudaStream_t st,
                     bool leaf_level = false) {
    ProfScope prof(c, nbytes, st, leaf_level);
    mxd::MsgJob j{};
    j.base = d_data; j.nbytes = nbytes; j.seg = seg;
    j.nmsg = nbytes ? (nbytes + seg - 1) / seg : 1;
    j.out = d_out; j.finalize = 1; j.one = 1;
    if (j.base == nullptr) j.base = reinterpret_cast<const uint8_t*>(d_out);   // empty message: any non-null base keeps the kernel in segment mode
    MXD_CUDA(mxd::launch_sha256(j, st));
    c->launches++; c->bytes_hashed += nbytes;
    return MXD_OK;
}

// digests of one tree level -> the next: groups of `fanout` digests
int enqueue_level(Core* c, const uint8_t* d_in, uint64_t n, uint64_t fanout, uint8_t* d_out, cudaStream_t st) {
    return enqueue_segments(c, d_in, n * 32, 32 * fanout, d_out, st);
}

// How many tree levels the leaf kernel computes itself for this tree when a piece is at least `avail` bytes long
// (0 = plain leaf digests, every level up to the chunk list its own launch: the default).
uint32_t fused_levels(const Tree& t, uint64_t avail) {
    if (!mxd::leaf_kernel_selected()) return 0;
    uint32_t f = mxd::leaf_fusable_levels((uint32_t)t.fanout, (uint32_t)t.klevel);
    while (f > 0 && t.leaf * ipow(t.fanout, f) > avail) --f;
    return f;
}

// blob bytes in device memory -> digests of tree level `fused` (one launch, leaves never touch DRAM when fused > 0)
int enqueue_leaves(Core* c, const Tree& t, uint32_t fused, const uint8_t* d_piece, uint64_t nbytes, uint8_t* d_out, cudaStream_t st) {
    const uint64_t n0 = nbytes ? (nbytes + t.leaf - 1) / t.leaf : 1;
    // default: the leaf level is an ordinary segment launch (k_sha256_lanes, or the two-warp chain kernel for the few
    // thousand leaves of one ring slot); k_tree_leaves only when an A/B knob asks for it
    if (!mxd::leaf_kernel_selected()) return enqueue_segments(c, d_piece, nbytes, t.leaf, d_out, st, /*leaf_level=*/true);
    ProfScope prof(c, nbytes, st);
    uint32_t* sched = nullptr;
    MXD_CUDA(cudaMallocAsync(&sched, mxd::leaf_sched_bytes(n0), st));
    mxd::LeafJob j{};
    j.base = d_piece ? d_piece : reinterpret_cast<const uint8_t*>(d_out);
    j.nbytes = nbytes; j.leaf = t.leaf; j.n0 = n0; j.fanout = (uint32_t)t.fanout; j.fused = fused;
    j.out = d_out; j.sched = sched; j.one = 1;
    cudaError_t e = mxd::launch_tree_leaves(j, st);
    cudaFreeAsync(sched, st);
    if (e != cudaSuccess) return fail(MXD_ERR_CUDA, std::string("launch_tree_leaves: ") + cudaGetErrorString(e));
    c->launches++; c->bytes_hashed += nbytes;
    return MXD_OK;
}

// digests of level `from` (n of them in d_in, clobbered as scratch) -> chunk digests (level k)
int enqueue_levels_to_chunks(Core* c, const Tree& t, uint32_t from, uint8_t* d_in, uint64_t n, uint8_t* d_chunks, cudaStream_t st) {
    if ((int)from >= t.klevel) return MXD_OK;     // the caller wrote level k straight into d_chunks
    const uint64_t n1 = (n + t.fanout - 1) / t.fanout;
    uint8_t* scratch = nullptr;
    if (t.klevel - (int)from > 1) MXD_CUDA(cudaMallocAsync(&scratch, n1 * 32, st));
    uint8_t* cur = d_in;
    int rc = MXD_OK;
    for (int lv = (int)from + 1; lv <= t.klevel && rc == MXD_OK; ++lv) {
        const uint64_t nn = (n + t.fanout - 1) / t.fanout;
        uint8_t* dst = (lv == t.klevel) ? d_chunks : ((cur == d_in) ? scratch : d_in);
        rc = enqueue_level(c, cur, n, t.fanout, dst, st);
        cur = dst; n = nn;
    }
    if (scratch) cudaFreeAsync(scratch, st);
    return rc;
}

// leaves -> chunk digests for one piece resident in device memory
int enqueue_tree_chunks(Core* c, const Tree& t, const uint8_t* d_piece, uint64_t nbytes, uint8_t* d_chunks, cudaStream_t st) {
    const uint64_t n0 = nbytes ? (nbytes + t.leaf - 1) / t.leaf : 1;
    const uint32_t fused = fused_levels(t, ~0ull);
    if ((int)fused == t.klevel) return enqueue_leaves(c, t, fused, d_piece, nbytes, d_chunks, st);
    const uint64_t span = ipow(t.fanout, fused);
    const uint64_t nf = (n0 + span - 1) / span;
    uint8_t* ws = nullptr;
    MXD_CUDA(cudaMallocAsync(&ws, nf * 32, st));
    int rc = enqueue_leaves(c, t, fused, d_piece, nbytes, ws, st);
    if (rc == MXD_OK) rc = enqueue_levels_to_chunks(c, t, fused, ws, nf, d_chunks, st);
    cudaFreeAsync(ws, st);
    return rc;
}

// levels above the chunk list, then the root message
int enqueue_tree_finish(Core* c, const Tree& t, const uint8_t* d_chunks, uint64_t nchunks, uint64_t size,
                        uint8_t* d_root, cudaStream_t st) {
    uint8_t* scratch = nullptr;
    MXD_CUDA(cudaMallocAsync(&scratch, mxd::tree_top_scratch_bytes(nchunks, (uint32_t)t.fanout), st));
    cudaError_t e = mxd::launch_tree_top(d_chunks, nchunks, (uint32_t)t.fanout, size, t.leaf, scratch, d_root, st);
    cudaFreeAsync(scratch, st);
    if (e != cudaSuccess) return fail(MXD_ERR_CUDA, std::string("launch_tree_top: ") + cudaGetErrorString(e));
    c->launches++;
    return MXD_OK;
}

// ---- slot timeline ---------------------------------------------------------------------------------------------
struct TraceSlot {
    Core* c; Core::TraceRec rec{}; bool on = false;
    TraceSlot(Core* core, int ordinal, int slot, uint64_t bytes, double fill_ms) : c(core) {
        if (!c->trace_on.load()) return;
        { std::lock_guard<std::mutex> lk(c->trace_mu); if (c->trace.size() >= (1u << 15)) return; }
        rec.ordinal = ordinal; rec.slot = slot; rec.bytes = bytes; rec.fill_ms = fill_ms;
        if (cudaEventCreate(&rec.c0) != cudaSuccess || cudaEventCreate(&rec.c1) != cudaSuccess ||
            cudaEventCreate(&rec.k0) != cudaSuccess || cudaEventCreate(&rec.k1) != cudaSuccess) return;
        on = true;
    }
    void commit() { if (on) { std::lock_guard<std::mutex> lk(c->trace_mu); c->trace.push_back(rec); } }
};

// Stream [0, nbytes) of `src` through device `d`'s ring and hash it as tree leaves of t.leaf bytes (with `fused`
// levels computed in the same kernel) into d_out.  H2D copies run on the copy stream, kernels on the compute
// stream; a slot is refilled only after the kernel that read it has finished, so copy k+1.. overlap kernel k.
struct RingCursor { uint64_t i = 0; };     // running slot index: lets consecutive blobs share one pipelined pass over the ring

int stream_leaves(Core* c, const CancelScope& cs, DevState* d, const Tree& t, uint32_t fused, const Source& src, uint64_t nbytes,
                  uint8_t* d_out, RingCursor* cur = nullptr) {
    RingCursor own;
    if (!cur) cur = &own;
    const uint64_t unit = t.leaf * ipow(t.fanout, fused);       // bytes under one output digest
    const uint64_t per_slot = (d->slot_bytes / unit) * unit;
    if (per_slot == 0) return fail(MXD_ERR_INVALID, "ring slot smaller than one leaf; raise ring_bytes");
    if (nbytes == 0) return enqueue_leaves(c, t, fused, nullptr, 0, d_out, d->compute);
    uint64_t off = 0;
    for (; off < nbytes; ++cur->i) {
        const uint64_t i = cur->i;
        if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
        const int s = (int)(i % kSlots);
        const uint64_t n = (nbytes - off < per_slot) ? nbytes - off : per_slot;
        if (i >= (uint64_t)kSlots) MXD_CUDA(cudaEventSynchronize(d->ev_done[s]));
        uint8_t* h_slot = d->h_ring + (uint64_t)s * d->slot_bytes;
        uint8_t* d_slot = d->d_ring + (uint64_t)s * d->slot_bytes;
        const uint8_t* from = nullptr;
        int rc = MXD_OK;
        const double f0 = c->trace_on.load() ? now_ms() : 0;
        { PhaseTimer pt("  fill slot"); rc = source_stage(c, src, off, n, h_slot, &from, d->pool); }
        if (rc != MXD_OK) return rc;
        TraceSlot tr(c, d->ordinal, s, n, c->trace_on.load() ? now_ms() - f0 : 0);
        if (tr.on) cudaEventRecord(tr.rec.c0, d->copy);
        MXD_CUDA(cudaMemcpyAsync(d_slot, from, n, cudaMemcpyHostToDevice, d->copy));
        if (tr.on) cudaEventRecord(tr.rec.c1, d->copy);
        MXD_CUDA(cudaEventRecord(d->ev_copied[s], d->copy));
        MXD_CUDA(cudaStreamWaitEvent(d->compute, d->ev_copied[s], 0));
        if (tr.on) cudaEventRecord(tr.rec.k0, d->compute);
        rc = enqueue_leaves(c, t, fused, d_slot, n, d_out + (off / unit) * 32, d->compute);
        if (rc != MXD_OK) return rc;
        if (tr.on) cudaEventRecord(tr.rec.k1, d->compute);
        tr.commit();
        MXD_CUDA(cudaEventRecord(d->ev_done[s], d->compute));
        rc = sink_pieces(src, off, n, from, d->pool);     // the tee runs while the copy engine and the SMs work on this slot
        if (rc != MXD_OK) return rc;
        c->h2d += n;
        off += n;
    }
    return MXD_OK;
}

// Stream [0, size) of `src` through device `d`'s pinned ring straight into the caller's device spans (`table`: the
// non-empty spans with their offsets in the concatenation, `d_table` its device copy) and hash the leaves of every slot
// from the spans with k_tree_leaves_extents, writing leaf digests to d_leaves (n0 * 32 bytes).  Slots hold whole
// leaves.  The H2D copies of a slot go on the copy stream, its kernel on the compute stream after them; the kernel never
// reads the pinned slot, so a slot is refilled as soon as its own copies are done.
int load_leaves(Core* c, const CancelScope& cs, DevState* d, const Tree& t, const Source& src, uint64_t size,
                const std::vector<mxd::DevExtent>& table, const mxd::DevExtent* d_table, uint8_t* d_leaves) {
    const uint64_t per_slot = (d->slot_bytes / t.leaf) * t.leaf;
    if (per_slot == 0) return fail(MXD_ERR_INVALID, "ring slot smaller than one leaf; raise ring_bytes");
    auto leaves = [&](uint64_t first, uint64_t count, uint64_t nbytes) -> int {
        ProfScope prof(c, nbytes, d->compute);
        mxd::ExtentLeafJob j{};
        j.ext = d_table; j.m = table.size(); j.size = size; j.leaf = t.leaf; j.first = first; j.n0 = count;
        j.out = d_leaves + first * 32; j.one = 1;
        MXD_CUDA(mxd::launch_tree_leaves_extents(j, d->compute));
        c->launches++; c->bytes_hashed += nbytes;
        return MXD_OK;
    };
    if (size == 0) return leaves(0, 1, 0);
    size_t e = 0;                  // first span that ends after `off`
    uint64_t off = 0;
    for (uint64_t i = 0; off < size; ++i) {
        if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
        const int s = (int)(i % kSlots);
        const uint64_t n = (size - off < per_slot) ? size - off : per_slot;
        if (i >= (uint64_t)kSlots) MXD_CUDA(cudaEventSynchronize(d->ev_copied[s]));
        uint8_t* h_slot = d->h_ring + (uint64_t)s * d->slot_bytes;
        const uint8_t* from = nullptr;
        const double f0 = c->trace_on.load() ? now_ms() : 0;
        int rc = source_stage(c, src, off, n, h_slot, &from, d->pool);
        if (rc != MXD_OK) return rc;
        TraceSlot tr(c, d->ordinal, s, n, c->trace_on.load() ? now_ms() - f0 : 0);
        if (tr.on) cudaEventRecord(tr.rec.c0, d->copy);
        for (size_t k = e; k < table.size() && table[k].start < off + n; ++k) {     // the pieces of the spans in this slot
            const uint64_t a = std::max(table[k].start, off), b = std::min(table[k].start + table[k].len, off + n);
            MXD_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(const_cast<void*>(table[k].ptr)) + (a - table[k].start), from + (a - off),
                                     b - a, cudaMemcpyHostToDevice, d->copy));
        }
        while (e < table.size() && table[e].start + table[e].len <= off + n) ++e;
        if (tr.on) cudaEventRecord(tr.rec.c1, d->copy);
        MXD_CUDA(cudaEventRecord(d->ev_copied[s], d->copy));
        MXD_CUDA(cudaStreamWaitEvent(d->compute, d->ev_copied[s], 0));
        if (tr.on) cudaEventRecord(tr.rec.k0, d->compute);
        rc = leaves(off / t.leaf, (n + t.leaf - 1) / t.leaf, n);
        if (rc != MXD_OK) return rc;
        if (tr.on) cudaEventRecord(tr.rec.k1, d->compute);
        tr.commit();
        c->h2d += n;
        off += n;
    }
    return MXD_OK;
}

// chunk digests of a host/file piece on one device; result left in device memory d_chunks
int stream_tree_chunks(Core* c, const CancelScope& cs, DevState* d, const Tree& t, const Source& src, uint64_t nbytes, uint8_t* d_chunks) {
    const uint64_t n0 = nbytes ? (nbytes + t.leaf - 1) / t.leaf : 1;
    const uint32_t fused = fused_levels(t, d->slot_bytes);
    const uint64_t span = ipow(t.fanout, fused);
    const uint64_t nf = (n0 + span - 1) / span;
    const bool direct = (int)fused == t.klevel;
    uint8_t* d_lvl = d_chunks;
    if (!direct) { PhaseTimer pt("alloc level digests"); MXD_CUDA(cudaMallocAsync(&d_lvl, nf * 32, d->compute)); }
    int rc;
    { PhaseTimer pt("stream_leaves (enqueue)"); rc = stream_leaves(c, cs, d, t, fused, src, nbytes, d_lvl); }
    if (rc == MXD_OK && !direct) rc = enqueue_levels_to_chunks(c, t, fused, d_lvl, nf, d_chunks, d->compute);
    if (rc != MXD_OK) cudaStreamSynchronize(d->copy);   // nothing may still be reading the caller's (pinned) memory
    cudaError_t e;
    { PhaseTimer pt("sync compute"); e = cudaStreamSynchronize(d->compute); }
    if (rc == MXD_OK && e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    if (!direct) cudaFreeAsync(d_lvl, d->compute);
    return rc;
}

// Chunk digests of a host/file blob using every device of the context: device g takes the
// contiguous chunk range [g*n/G, (g+1)*n/G) (sequential reads per device, no data-path
// collective).  Results land in host memory `out` (nchunks*32).
int host_tree_chunks_all(Core* c, const CancelScope& cs, const Tree& t, const Source& src, uint64_t nbytes, uint8_t* out) {
    const uint64_t chunk = t.chunk;
    const uint64_t nchunks = nbytes ? (nbytes + chunk - 1) / chunk : 1;
    const int G = (int)std::min<uint64_t>(c->devs.size(), nchunks);
    std::vector<int> rcs(G, MXD_OK);
    std::vector<std::string> errs(G);
    auto work = [&](int g) {
        DevState* d = c->devs[g];
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard guard(d->ordinal);
        const uint64_t c0 = nchunks * g / G, c1 = nchunks * (g + 1) / G;
        const uint64_t b0 = c0 * chunk, b1 = std::min<uint64_t>(c1 * chunk, nbytes);
        Source piece = src;
        if (piece.fd >= 0) piece.base += b0; else piece.mem += b0;
        piece.sink_base += b0;
        FileMapGuard fm; fm.attach(&piece, b1 - b0);        // unmapped after stream_tree_chunks has synchronised
        uint8_t* d_chunks = nullptr;
        cudaError_t e = cudaMallocAsync(&d_chunks, (c1 - c0) * 32, d->compute);
        if (e != cudaSuccess) { rcs[g] = MXD_ERR_CUDA; errs[g] = cudaGetErrorString(e); return; }
        int rc = stream_tree_chunks(c, cs, d, t, piece, b1 - b0, d_chunks);
        if (rc == MXD_OK) {
            PhaseTimer pt("chunk digests D2H");
            e = cudaMemcpyAsync(out + c0 * 32, d_chunks, (c1 - c0) * 32, cudaMemcpyDeviceToHost, d->compute);
            if (e == cudaSuccess) e = cudaStreamSynchronize(d->compute);
            if (e != cudaSuccess) { rc = MXD_ERR_CUDA; fail(rc, cudaGetErrorString(e)); }
            c->d2h += (c1 - c0) * 32;
        }
        cudaFreeAsync(d_chunks, d->compute);
        rcs[g] = rc;
        if (rc != MXD_OK) errs[g] = last_error();
    };
    if (G == 1) {
        work(0);
    } else {
        std::vector<std::thread> th;
        for (int g = 0; g < G; ++g) th.emplace_back(work, g);
        for (auto& t2 : th) t2.join();
    }
    for (int g = 0; g < G; ++g)
        if (rcs[g] != MXD_OK) return fail(rcs[g], errs[g]);
    return MXD_OK;
}

// Tree roots of many files on one device, back to back through the ring: the copy engine and the SMs never drain between
// files (a per-file call pays pipeline fill and a sync per file: 128 MB files would run at less than half the rate).
// Everything of a file after its last slot (levels, root, D2H of the root) is stream-ordered behind it; one sync at the end.
struct TreeFileItem { const char* path; uint8_t* root; uint64_t size = 0; int status = MXD_OK; std::string error; };

int tree_files_on_device(Core* c, const CancelScope& cs, DevState* d, const Tree& t, std::vector<TreeFileItem*>& items) {
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard guard(d->ordinal);
    uint8_t* h_roots = nullptr;
    MXD_CUDA(cudaHostAlloc(&h_roots, 32 * std::max<size_t>(items.size(), 1), cudaHostAllocPortable));
    RingCursor cur;
    int rc = MXD_OK;
    const uint32_t fused = fused_levels(t, d->slot_bytes);
    const uint64_t span = ipow(t.fanout, fused);
    std::vector<std::unique_ptr<FileMapGuard>> maps;
    for (size_t k = 0; k < items.size() && rc == MXD_OK; ++k) {
        if (maps.size() > 64) maps.erase(maps.begin(), maps.begin() + 32);     // staged bytes of old files are long since copied
        TreeFileItem& it = *items[k];
        int fd = open(it.path, O_RDONLY | O_CLOEXEC);
        struct stat st;
        if (fd < 0 || fstat(fd, &st) != 0 || S_ISDIR(st.st_mode)) {
            it.status = MXD_ERR_IO; it.error = std::string(fd < 0 ? "open " : "read ") + it.path + ": " + (fd >= 0 && S_ISDIR(st.st_mode) ? "is a directory" : strerror(errno));
            if (fd >= 0) close(fd);
            continue;
        }
        it.size = (uint64_t)st.st_size;
        const uint64_t n0 = it.size ? (it.size + t.leaf - 1) / t.leaf : 1, nf = (n0 + span - 1) / span;
        const uint64_t nchunks = it.size ? (it.size + t.chunk - 1) / t.chunk : 1;
        uint8_t *d_lvl = nullptr, *d_chunks = nullptr;      // [level digests][chunk digests][root]
        cudaError_t e = cudaMallocAsync(&d_lvl, nf * 32, d->compute);
        if (e == cudaSuccess) e = cudaMallocAsync(&d_chunks, nchunks * 32 + 32, d->compute);
        if (e != cudaSuccess) { close(fd); rc = fail(MXD_ERR_CUDA, std::string("cudaMallocAsync: ") + cudaGetErrorString(e)); break; }
        Source src; src.fd = fd;
        maps.emplace_back(new FileMapGuard()); maps.back()->attach(&src, it.size);   // the fills of this file are done when stream_leaves returns,
        int r = stream_leaves(c, cs, d, t, fused, src, it.size, d_lvl, &cur);         // but keep it simple: unmap after the final sync
        close(fd);
        if (r == MXD_OK) {
            if ((int)fused == t.klevel) e = cudaMemcpyAsync(d_chunks, d_lvl, nchunks * 32, cudaMemcpyDeviceToDevice, d->compute);
            else r = enqueue_levels_to_chunks(c, t, fused, d_lvl, nf, d_chunks, d->compute);
        }
        if (r == MXD_OK && e == cudaSuccess) r = enqueue_tree_finish(c, t, d_chunks, nchunks, it.size, d_chunks + nchunks * 32, d->compute);
        if (r == MXD_OK && e == cudaSuccess) e = cudaMemcpyAsync(h_roots + 32 * k, d_chunks + nchunks * 32, 32, cudaMemcpyDeviceToHost, d->compute);
        cudaFreeAsync(d_lvl, d->compute); cudaFreeAsync(d_chunks, d->compute);
        if (r == MXD_ERR_CANCELED || r == MXD_ERR_CUDA || e != cudaSuccess) { rc = (e != cudaSuccess) ? fail(MXD_ERR_CUDA, cudaGetErrorString(e)) : r; break; }
        if (r != MXD_OK) { it.status = r; it.error = last_error(); }      // I/O trouble with this file only
        c->d2h += 32;
    }
    cudaError_t e = cudaStreamSynchronize(d->compute);
    cudaStreamSynchronize(d->copy);
    if (rc == MXD_OK && e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    if (rc == MXD_OK) for (size_t k = 0; k < items.size(); ++k) if (items[k]->status == MXD_OK) memcpy(items[k]->root, h_roots + 32 * k, 32);
    cudaFreeHost(h_roots);
    return rc;
}

// upper levels + root from a host-resident chunk list (tiny: 32 B per chunk)
int host_tree_finish(Core* c, DevState* d, const Tree& t, const uint8_t* chunks, uint64_t nchunks, uint64_t size,
                     uint8_t root[32]) {
    PhaseTimer pt("tree finish (levels + root)");
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard guard(d->ordinal);
    uint8_t* d_buf = nullptr;
    MXD_CUDA(cudaMallocAsync(&d_buf, nchunks * 32 + 32, d->compute));
    int rc = MXD_OK;
    cudaError_t e = cudaMemcpyAsync(d_buf, chunks, nchunks * 32, cudaMemcpyHostToDevice, d->compute);
    if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, cudaGetErrorString(e));
    if (rc == MXD_OK) rc = enqueue_tree_finish(c, t, d_buf, nchunks, size, d_buf + nchunks * 32, d->compute);
    if (rc == MXD_OK) {
        e = cudaMemcpyAsync(root, d_buf + nchunks * 32, 32, cudaMemcpyDeviceToHost, d->compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(d->compute);
        if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, cudaGetErrorString(e));
        c->h2d += nchunks * 32; c->d2h += 32;
    } else {
        cudaStreamSynchronize(d->compute);
    }
    cudaFreeAsync(d_buf, d->compute);
    return rc;
}

bool handle_ok(const mxd_ctx* h) { return h != nullptr && h->core != nullptr; }

}  // namespace
}  // namespace mxdi

#ifdef MXD_MOCK_CUDA
namespace mxd {
// Only in the CPU test double (tests/mock), which compiles the host sources of this library with its own kernel
// launchers and has none for k_tree_leaves_extents: there the leaf level is the concatenation gathered into one
// buffer and hashed as uniform leaf-sized segments through launch_sha256, so the host logic of
// mxd_dev_tree_digest_extents runs unchanged.  The CUDA build never compiles this.
cudaError_t launch_tree_leaves_extents(const ExtentLeafJob& j, cudaStream_t st) {
    if (j.n0 == 0 || (j.size != 0 && (j.m == 0 || j.ext == nullptr)) || j.out == nullptr) return cudaErrorInvalidValue;
    if (j.first != 0 && j.first * j.leaf >= j.size) return cudaErrorInvalidValue;
    uint8_t* cat = nullptr;
    cudaError_t e = cudaMallocAsync(&cat, j.size ? j.size : 1, st);
    for (uint64_t i = 0; e == cudaSuccess && i < j.m; ++i)
        e = cudaMemcpyAsync(cat + j.ext[i].start, j.ext[i].ptr, j.ext[i].len, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) {
        const uint64_t skip = j.first * j.leaf;     // leaves [first, first + n0): the segments from byte first * leaf on
        MsgJob m{};
        m.base = cat + skip; m.nbytes = j.size - skip; m.seg = j.leaf; m.nmsg = j.n0; m.out = j.out; m.finalize = 1; m.one = j.one;
        e = launch_sha256(m, st);
    }
    if (cat) cudaFreeAsync(cat, st);
    return e;
}
}  // namespace mxd
#endif

using namespace mxdi;

// =================================================================================================
extern "C" {

int mxd_abi_version(void) { return MXD_ABI_VERSION; }

const char* mxd_strerror(int status) {
    switch (status) {
        case MXD_OK: return "ok";
        case MXD_ERR_INVALID: return "invalid argument";
        case MXD_ERR_NO_DEVICE: return "no CUDA device available (modelx-b200 has no CPU fallback)";
        case MXD_ERR_CUDA: return "CUDA error";
        case MXD_ERR_IO: return "I/O error";
        case MXD_ERR_NOMEM: return "out of memory";
        case MXD_ERR_CANCELED: return "canceled";
        case MXD_ERR_DIV_ZERO: return "integer divide by zero (calcParts with 0 parts)";
        default: return "unknown status";
    }
}

const char* mxd_last_error(void) { return last_error().c_str(); }

int mxd_prof_enable(mxd_ctx* h, int on) {
    if (!handle_ok(h)) return fail(MXD_ERR_INVALID, "prof_enable: null");
    h->core->prof_on.store(on ? 1 : 0);
    return MXD_OK;
}

int mxd_prof_read(mxd_ctx* h, double* kernel_ms, uint64_t* launches, uint64_t* bytes) {
    if (!handle_ok(h)) return fail(MXD_ERR_INVALID, "prof_read: null");
    Core* c = h->core;
    std::vector<Core::ProfRec> recs;
    { std::lock_guard<std::mutex> lk(c->prof_mu); recs.swap(c->prof); }
    double ms = 0; uint64_t nb = 0;
    int rc = MXD_OK;
    for (auto& r : recs) {
        DeviceGuard guard(r.ordinal);
        float t = 0;
        cudaError_t e = cudaEventSynchronize(r.b);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&t, r.a, r.b);
        if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("prof_read: ") + cudaGetErrorString(e));
        ms += t; nb += r.bytes;
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    if (kernel_ms) *kernel_ms = ms;
    if (launches) *launches = recs.size();
    if (bytes) *bytes = nb;
    return rc;
}

int mxd_trace_enable(mxd_ctx* h, int on) {
    if (!handle_ok(h)) return fail(MXD_ERR_INVALID, "trace_enable: null");
    h->core->trace_on.store(on ? 1 : 0);
    return MXD_OK;
}

int mxd_trace_dump(mxd_ctx* h, const char* path) {
    if (!handle_ok(h) || !path) return fail(MXD_ERR_INVALID, "trace_dump: bad arguments");
    Core* c = h->core;
    std::vector<Core::TraceRec> recs;
    { std::lock_guard<std::mutex> lk(c->trace_mu); recs.swap(c->trace); }
    FILE* f = fopen(path, "w");
    if (!f) return fail(MXD_ERR_IO, std::string("open ") + path + ": " + strerror(errno));
    fprintf(f, "device,slot,bytes,host_fill_ms,h2d_start_ms,h2d_end_ms,kernel_start_ms,kernel_end_ms\n");
    int rc = MXD_OK;
    std::vector<cudaEvent_t> origin(64, nullptr);      // per device: the first record's copy start
    for (auto& r : recs) {
        DeviceGuard guard(r.ordinal);
        if (r.ordinal >= 0 && r.ordinal < 64 && !origin[r.ordinal]) origin[r.ordinal] = r.c0;
        cudaEvent_t o = (r.ordinal >= 0 && r.ordinal < 64) ? origin[r.ordinal] : r.c0;
        float c0 = 0, c1 = 0, k0 = 0, k1 = 0;
        cudaError_t e = cudaEventSynchronize(r.k1);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&c0, o, r.c0);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&c1, o, r.c1);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&k0, o, r.k0);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&k1, o, r.k1);
        if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("trace_dump: ") + cudaGetErrorString(e));
        fprintf(f, "%d,%d,%llu,%.3f,%.3f,%.3f,%.3f,%.3f\n", r.ordinal, r.slot, (unsigned long long)r.bytes, r.fill_ms, c0, c1, k0, k1);
    }
    for (auto& r : recs) { DeviceGuard guard(r.ordinal); cudaEventDestroy(r.c0); cudaEventDestroy(r.c1); cudaEventDestroy(r.k0); cudaEventDestroy(r.k1); }
    fclose(f);
    return rc;
}

int mxd_open(mxd_ctx** out, const int* devices, int ndev, uint64_t ring_bytes) {
    if (!out || ndev < 0 || (ndev > 0 && !devices)) return fail(MXD_ERR_INVALID, "mxd_open: bad arguments");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        return fail(MXD_ERR_NO_DEVICE, std::string("cudaGetDeviceCount: ") + (e == cudaSuccess ? "0 devices" : cudaGetErrorString(e)));
    }
    std::vector<int> ords;
    if (ndev == 0) for (int i = 0; i < count; ++i) ords.push_back(i);
    else for (int i = 0; i < ndev; ++i) {
        if (devices[i] < 0 || devices[i] >= count) return fail(MXD_ERR_INVALID, "mxd_open: device ordinal out of range");
        ords.push_back(devices[i]);
    }
    if (const char* env = getenv("MXD_RING_BYTES")) { uint64_t v = strtoull(env, nullptr, 10); if (v) ring_bytes = v; }
    if (ring_bytes == 0) ring_bytes = kDefaultRingBytes;
    uint64_t slot = (ring_bytes / kSlots) & ~((1ull << 20) - 1);
    if (slot < (1ull << 20)) slot = 1ull << 20;

    auto* c = new Core();
    auto* h = new mxd_ctx();
    h->core = c;
    // the digest service keeps at most this many files open at once (the reference holds 3: push.go:27)
    struct rlimit rl;
    if (getrlimit(RLIMIT_NOFILE, &rl) == 0 && rl.rlim_cur != RLIM_INFINITY)
        c->fd_cap = (int)std::max<long>(8, std::min<long>(4096, (long)rl.rlim_cur / 2 - 32));
    else c->fd_cap = 4096;
    if (const char* env = getenv("MXD_MAX_OPEN_FILES")) { int v = atoi(env); if (v > 0) c->fd_cap = v; }
    int prev = -1; cudaGetDevice(&prev);
    // slot-filler threads per device: MXD_STAGE_THREADS, default min(16, hw threads / devices), at least 1
    // (page-cache pread runs at a few GB/s per thread; beyond ~16 threads a tmpfs file reads slower, not faster)
    int stage_threads = 0;
    if (const char* env = getenv("MXD_STAGE_THREADS")) stage_threads = atoi(env);
    if (stage_threads <= 0) {
        // CPUs this process may really use: affinity mask, capped by a cgroup CPU quota (the bench container has 128
        // CPUs visible and a quota of 16), shared with the other ranks of a torchrun launch on the same node
        unsigned usable = std::thread::hardware_concurrency();
        cpu_set_t aff;
        if (sched_getaffinity(0, sizeof aff, &aff) == 0 && CPU_COUNT(&aff) > 0) usable = (unsigned)CPU_COUNT(&aff);
        if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
            char q[64] = {0}; unsigned long period = 0;
            if (fscanf(f, "%63s %lu", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
                const unsigned long quota = strtoul(q, nullptr, 10) / period;
                if (quota > 0 && quota < usable) usable = (unsigned)quota;
            }
            fclose(f);
        }
        unsigned sharers = (unsigned)ords.size();
        if (const char* lw = getenv("LOCAL_WORLD_SIZE")) { const int v = atoi(lw); if (v > 0) sharers = std::max<unsigned>(sharers, (unsigned)v * (unsigned)ords.size()); }
        stage_threads = (int)std::min<unsigned>(16, std::max<unsigned>(2, usable / std::max(1u, sharers)));
    }
    for (int ord : ords) {
        auto* d = new DevState();
        d->ordinal = ord; d->slot_bytes = slot;
        c->devs.push_back(d);
        if ((e = cudaSetDevice(ord)) != cudaSuccess) break;
        LocalCpuScope numa(ord);     // the pool's threads inherit this affinity; the pinned ring is first-touched here
        d->pool = new StagePool(stage_threads - 1);
        if ((e = cudaStreamCreateWithFlags(&d->compute, cudaStreamNonBlocking)) != cudaSuccess) break;
        if ((e = cudaStreamCreateWithFlags(&d->copy, cudaStreamNonBlocking)) != cudaSuccess) break;
        if ((e = cudaHostAlloc(&d->h_ring, slot * kSlots, cudaHostAllocPortable)) != cudaSuccess) break;
        if ((e = cudaMalloc(&d->d_ring, slot * kSlots)) != cudaSuccess) break;
        for (int s = 0; s < kSlots && e == cudaSuccess; ++s) {
            e = cudaEventCreateWithFlags(&d->ev_copied[s], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&d->ev_done[s], cudaEventDisableTiming);
        }
        if (e != cudaSuccess) break;
        // keep stream-ordered workspace allocations cached instead of returning them to the OS
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, ord) == cudaSuccess) {
            uint64_t keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    }
    if (prev >= 0) cudaSetDevice(prev);
    if (e != cudaSuccess) {
        int rc = fail(MXD_ERR_CUDA, std::string("mxd_open: ") + cudaGetErrorString(e));
        mxd_close(h);
        return rc;
    }
    *out = h;
    return MXD_OK;
}

void mxd_close(mxd_ctx* h) {
    if (!h) return;
    if (h->parent) { mxd_op_end(h); return; }     // closing an operation handle ends the operation only
    Core* c = h->core;
    int prev = -1; cudaGetDevice(&prev);
    for (DevState* d : c->devs) {
        if (d->ordinal >= 0) cudaSetDevice(d->ordinal);
        svc_destroy(d);
        if (d->compute) { cudaStreamSynchronize(d->compute); cudaStreamDestroy(d->compute); }
        if (d->copy) { cudaStreamSynchronize(d->copy); cudaStreamDestroy(d->copy); }
        for (int s = 0; s < kSlots; ++s) {
            if (d->ev_copied[s]) cudaEventDestroy(d->ev_copied[s]);
            if (d->ev_done[s]) cudaEventDestroy(d->ev_done[s]);
        }
        if (d->h_ring) cudaFreeHost(d->h_ring);
        if (d->d_ring) cudaFree(d->d_ring);
        delete d->pool;
        delete d;
    }
    if (prev >= 0) cudaSetDevice(prev);
    delete c;
    delete h;
}

int mxd_op_begin(mxd_ctx* parent, mxd_ctx** op) {
    if (!handle_ok(parent) || !op) return fail(MXD_ERR_INVALID, "op_begin: bad arguments");
    auto* h = new mxd_ctx();
    h->core = parent->core;
    h->parent = parent->parent ? parent->parent : parent;
    h->core->live_ops++;
    *op = h;
    return MXD_OK;
}

void mxd_op_end(mxd_ctx* op) {
    if (!op || !op->parent) return;
    op->core->live_ops--;
    delete op;
}

int mxd_device_count(const mxd_ctx* h) { return handle_ok(h) ? (int)h->core->devs.size() : 0; }

void mxd_cancel(mxd_ctx* h) {
    if (!handle_ok(h)) return;
    if (h->parent) h->canceled.store(1);          // this operation only, and for good
    else h->core->cancel_gen++;                   // every call in flight on the context right now; later calls are unaffected
}
void mxd_reset_cancel(mxd_ctx* h) { if (handle_ok(h)) h->canceled.store(0); }
int mxd_is_canceled(const mxd_ctx* h) { return handle_ok(h) && h->canceled.load() ? 1 : 0; }

int mxd_get_stats(const mxd_ctx* h, mxd_stats* out) {
    if (!handle_ok(h) || !out) return fail(MXD_ERR_INVALID, "mxd_get_stats: null");
    const Core* c = h->core;
    memset(out, 0, sizeof *out);
    out->kernel_launches = mxd::kernel_launch_count(); out->bytes_hashed = c->bytes_hashed.load();
    out->h2d_bytes = c->h2d.load(); out->d2h_bytes = c->d2h.load();
    out->src_bytes_read = c->src_read.load();
    out->open_files = (uint64_t)std::max(0, c->open_fds.load());
    return MXD_OK;
}

// ---- integer split: extension_s3.go:99-112, store_s3.go:198-203,273-279 --------------------------
int mxd_calc_parts(int64_t total, int64_t partscount, mxd_part* out) {
    if (partscount == 0) return fail(MXD_ERR_DIV_ZERO, "calcParts: partscount == 0 (reference panics: integer divide by zero)");
    if (partscount < 0 || !out) return fail(MXD_ERR_INVALID, "calcParts: negative part count");
    const int64_t partsize = total / partscount;
    for (int64_t i = 0; i < partscount; ++i) {
        out[i].offset = i * partsize;
        out[i].length = (i == partscount - 1) ? total - out[i].offset : partsize;
    }
    return MXD_OK;
}

int64_t mxd_server_part_count(int64_t size, int force_multipart) {
    const int64_t kThreshold = 5ll << 30;   // MultiPartUploadThreshold
    const int64_t kDefaultParts = 3;        // DefaultPartCount
    if (!force_multipart && size <= kThreshold) return 1;
    int64_t count = size / kThreshold;
    if (count == 0) return kDefaultParts;
    return (size % kThreshold) ? count + 1 : count;
}

// ---- routing advice ------------------------------------------------------------------------------------------
// A whole-file SHA-256 is one serial chain: one GPU lane is an order of magnitude slower than one SHA-NI core, and the
// reference hashes 3 files at a time (push.go:27).  The GPU wins only through width.  Model (rates below): GPU time = max(longest blob / chain rate, total / PCIe rate) + launch overhead;
// CPU time = max(longest blob / core rate, total / (3 cores)).
int mxd_batch_pays_off(uint64_t n_blobs, uint64_t total_bytes, uint64_t max_blob_bytes) {
    if (n_blobs == 0) return 0;
    if (max_blob_bytes == 0 || max_blob_bytes > total_bytes) max_blob_bytes = (total_bytes + n_blobs - 1) / n_blobs;
    const double chain = 0.085e9, pcie = 45e9, core = 1.4e9, cpu_threads = 3;
    const double gpu_s = std::max((double)max_blob_bytes / chain, (double)total_bytes / pcie) + 0.002;
    const double cpu_s = std::max((double)max_blob_bytes / core, (double)total_bytes / (core * cpu_threads));
    return gpu_s < cpu_s ? 1 : 0;
}

// ---- digest strings -------------------------------------------------------------------------------
void mxd_digest_string(const uint8_t d[32], char out[72]) {
    static const char* hex = "0123456789abcdef";
    memcpy(out, "sha256:", 7);
    for (int i = 0; i < 32; ++i) { out[7 + 2 * i] = hex[d[i] >> 4]; out[8 + 2 * i] = hex[d[i] & 15]; }
    out[71] = 0;
}

int mxd_digest_parse(const char* s, uint8_t out[32]) {
    if (!s || strncmp(s, "sha256:", 7) != 0 || strlen(s) != 71) return fail(MXD_ERR_INVALID, "digest: want sha256:<64 lower hex>");
    for (int i = 0; i < 32; ++i) {
        int v = 0;
        for (int k = 0; k < 2; ++k) {
            const char ch = s[7 + 2 * i + k];
            int x = (ch >= '0' && ch <= '9') ? ch - '0' : (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : -1;
            if (x < 0) return fail(MXD_ERR_INVALID, "digest: invalid hex (go-digest accepts lower case only)");
            v = v * 16 + x;
        }
        if (out) out[i] = (uint8_t)v;
    }
    return MXD_OK;
}

// ---- tree ---------------------------------------------------------------------------------------------
int mxd_tree_shape(uint64_t size, const mxd_tree_params* tp, uint64_t* counts, int max_levels, int* chunk_level) {
    Tree t;
    if (!tree_resolve(tp, &t) || !counts || max_levels < 2) return fail(MXD_ERR_INVALID, "tree: chunk must be leaf * fanout^k (k >= 1), leaf a multiple of 64, fanout >= 2");
    uint64_t n = size ? (size + t.leaf - 1) / t.leaf : 1;
    int lv = 0;
    counts[lv++] = n;
    while (lv <= t.klevel || n > 1) {
        if (lv >= max_levels) return fail(MXD_ERR_INVALID, "tree: too many levels for counts[]");
        n = (n + t.fanout - 1) / t.fanout;
        counts[lv++] = n;
    }
    if (chunk_level) *chunk_level = t.klevel;
    return lv;
}

#define DEV_ARGS_OK(h, dev) (handle_ok(h) && (dev) >= 0 && (dev) < (int)(h)->core->devs.size())
// The kernels store digests as uint4 and k_tree_top reads digests as 32-bit words; spans are read as 8-byte fields.
static bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

int mxd_dev_sha256_segments(mxd_ctx* h, int dev, const void* d_data, uint64_t nbytes, uint64_t seg, void* d_out, void* stream) {
    if (!DEV_ARGS_OK(h, dev) || seg == 0 || !d_out || !aligned_to(d_out, 16) || (nbytes && !d_data))
        return fail(MXD_ERR_INVALID, "dev_sha256_segments: bad arguments");
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    return enqueue_segments(h->core, static_cast<const uint8_t*>(d_data), nbytes, seg, static_cast<uint8_t*>(d_out), (cudaStream_t)stream);
}

int mxd_dev_sha256_batch(mxd_ctx* h, int dev, const mxd_span* d_spans, uint64_t n, void* d_out, void* stream) {
    if (!DEV_ARGS_OK(h, dev) || (n && (!d_spans || !d_out)) || !aligned_to(d_spans, 8) || !aligned_to(d_out, 16))
        return fail(MXD_ERR_INVALID, "dev_sha256_batch: bad arguments");
    if (n == 0) return MXD_OK;
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    mxd::MsgJob j{};
    j.spans = d_spans; j.nmsg = n; j.out = static_cast<uint8_t*>(d_out); j.finalize = 1; j.one = 1;
    MXD_CUDA(mxd::launch_sha256(j, (cudaStream_t)stream));
    h->core->launches++;
    return MXD_OK;
}

int mxd_dev_tree_chunks(mxd_ctx* h, int dev, const void* d_piece, uint64_t nbytes, const mxd_tree_params* tp,
                        void* d_chunk_digests, void* stream) {
    Tree t;
    if (!DEV_ARGS_OK(h, dev) || !tree_resolve(tp, &t) || !d_chunk_digests || !aligned_to(d_chunk_digests, 16) || (nbytes && !d_piece))
        return fail(MXD_ERR_INVALID, "dev_tree_chunks: bad arguments");
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    return enqueue_tree_chunks(h->core, t, static_cast<const uint8_t*>(d_piece), nbytes, static_cast<uint8_t*>(d_chunk_digests),
                               (cudaStream_t)stream);
}

int mxd_dev_tree_finish(mxd_ctx* h, int dev, const void* d_chunk_digests, uint64_t nchunks, uint64_t size,
                        const mxd_tree_params* tp, void* d_root, void* stream) {
    Tree t;
    if (!DEV_ARGS_OK(h, dev) || !tree_resolve(tp, &t) || !d_chunk_digests || !d_root || nchunks == 0 ||
        !aligned_to(d_chunk_digests, 16) || !aligned_to(d_root, 16))
        return fail(MXD_ERR_INVALID, "dev_tree_finish: bad arguments");
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    return enqueue_tree_finish(h->core, t, static_cast<const uint8_t*>(d_chunk_digests), nchunks, size,
                               static_cast<uint8_t*>(d_root), (cudaStream_t)stream);
}

int mxd_dev_tree_digest(mxd_ctx* h, int dev, const void* d_data, uint64_t size, const mxd_tree_params* tp,
                        void* d_chunk_digests, void* d_root, void* stream) {
    Tree t;
    if (!DEV_ARGS_OK(h, dev) || !tree_resolve(tp, &t) || !d_root || !aligned_to(d_root, 16) || !aligned_to(d_chunk_digests, 16) ||
        (size && !d_data))
        return fail(MXD_ERR_INVALID, "dev_tree_digest: bad arguments");
    Core* c = h->core;
    DeviceGuard guard(c->devs[dev]->ordinal);
    cudaStream_t st = (cudaStream_t)stream;
    const uint64_t nchunks = size ? (size + t.chunk - 1) / t.chunk : 1;
    uint8_t* chunks = static_cast<uint8_t*>(d_chunk_digests);
    uint8_t* owned = nullptr;
    if (!chunks) { MXD_CUDA(cudaMallocAsync(&owned, nchunks * 32, st)); chunks = owned; }
    int rc = enqueue_tree_chunks(c, t, static_cast<const uint8_t*>(d_data), size, chunks, st);
    if (rc == MXD_OK) rc = enqueue_tree_finish(c, t, chunks, nchunks, size, static_cast<uint8_t*>(d_root), st);
    if (owned) cudaFreeAsync(owned, st);
    return rc;
}

int mxd_dev_tree_digest_extents(mxd_ctx* h, int dev, const mxd_span* extents, uint64_t n, const mxd_tree_params* tp,
                                void* d_chunk_digests, void* d_root, void* stream) {
    Tree t;
    if (!DEV_ARGS_OK(h, dev) || !tree_resolve(tp, &t) || (n && !extents) || !d_root || !aligned_to(d_root, 16) ||
        !aligned_to(d_chunk_digests, 16))
        return fail(MXD_ERR_INVALID, "dev_tree_digest_extents: bad arguments");
    // the device table: non-empty extents in order, each with its offset in the concatenation
    std::vector<mxd::DevExtent> table;
    uint64_t size = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (extents[i].len == 0) continue;
        if (!extents[i].ptr) return fail(MXD_ERR_INVALID, "dev_tree_digest_extents: extent " + std::to_string(i) + " is NULL with a nonzero length");
        if (extents[i].len > ~0ull - size) return fail(MXD_ERR_INVALID, "dev_tree_digest_extents: total length overflows 64 bits");
        table.push_back({extents[i].ptr, extents[i].len, size});
        size += extents[i].len;
    }
    Core* c = h->core;
    DeviceGuard guard(c->devs[dev]->ordinal);
    cudaStream_t st = (cudaStream_t)stream;
    const uint64_t nchunks = size ? (size + t.chunk - 1) / t.chunk : 1;
    const uint64_t n0 = size ? (size + t.leaf - 1) / t.leaf : 1;
    uint8_t* chunks = static_cast<uint8_t*>(d_chunk_digests);
    uint8_t* owned = nullptr;
    mxd::DevExtent* d_table = nullptr;
    uint8_t* ws = nullptr;
    if (!chunks) { MXD_CUDA(cudaMallocAsync(&owned, nchunks * 32, st)); chunks = owned; }
    int rc = MXD_OK;
    cudaError_t e = cudaMallocAsync(&ws, n0 * 32, st);
    if (e == cudaSuccess && !table.empty()) {
        e = cudaMallocAsync(&d_table, table.size() * sizeof(mxd::DevExtent), st);
        // From pageable memory, cudaMemcpyAsync returns only after the source has been staged, so `table` (and the
        // caller's array) may go away when this call returns.
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(mxd::DevExtent), cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("dev_tree_digest_extents: ") + cudaGetErrorString(e));
    if (rc == MXD_OK) {
        ProfScope prof(c, size, st);
        mxd::ExtentLeafJob j{};
        j.ext = d_table; j.m = table.size(); j.size = size; j.leaf = t.leaf; j.n0 = n0; j.out = ws; j.one = 1;
        e = mxd::launch_tree_leaves_extents(j, st);
        if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("launch_tree_leaves_extents: ") + cudaGetErrorString(e));
        else { c->launches++; c->bytes_hashed += size; }
    }
    if (rc == MXD_OK) rc = enqueue_levels_to_chunks(c, t, 0, ws, n0, chunks, st);
    if (rc == MXD_OK) rc = enqueue_tree_finish(c, t, chunks, nchunks, size, static_cast<uint8_t*>(d_root), st);
    if (d_table) cudaFreeAsync(d_table, st);
    if (ws) cudaFreeAsync(ws, st);
    if (owned) cudaFreeAsync(owned, st);
    return rc;
}

int mxd_dev_compare(mxd_ctx* h, int dev, const void* d_got, const void* d_want, uint64_t n, void* d_ok, void* stream) {
    if (!DEV_ARGS_OK(h, dev) || (n && (!d_got || !d_want || !d_ok))) return fail(MXD_ERR_INVALID, "dev_compare: bad arguments");
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    MXD_CUDA(mxd::launch_compare(static_cast<const uint8_t*>(d_got), static_cast<const uint8_t*>(d_want), n,
                                 static_cast<uint8_t*>(d_ok), (cudaStream_t)stream));
    if (n) h->core->launches++;
    return MXD_OK;
}

int mxd_dev_gen_fill(mxd_ctx* h, int dev, void* d_dst, uint64_t offset, uint64_t n, uint64_t seed, void* stream) {
    if (!DEV_ARGS_OK(h, dev) || (n && !d_dst) || !aligned_to(d_dst, 8) || ((offset | n) & 7u))
        return fail(MXD_ERR_INVALID, "dev_gen_fill: bad arguments");
    DeviceGuard guard(h->core->devs[dev]->ordinal);
    MXD_CUDA(mxd::launch_gen_fill(d_dst, offset, n, seed, (cudaStream_t)stream));
    if (n) h->core->launches++;
    return MXD_OK;
}

int mxd_tree_chunks(mxd_ctx* h, const void* piece, uint64_t nbytes, const mxd_tree_params* tp, uint8_t* out) {
    Tree t;
    if (!handle_ok(h) || !tree_resolve(tp, &t) || !out || (nbytes && !piece)) return fail(MXD_ERR_INVALID, "tree_chunks: bad arguments");
    Core* c = h->core;
    const CancelScope cs(h);
    if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
    const uint64_t nchunks = nbytes ? (nbytes + t.chunk - 1) / t.chunk : 1;
    int ord = -1;
    const MemKind kind = classify(piece, &ord);
    if (kind == MemKind::Device) {
        const int di = dev_index_of(c, ord);
        if (di < 0) return fail(MXD_ERR_INVALID, "tree_chunks: data lives on a device this context does not drive");
        DevState* d = c->devs[di];
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard guard(d->ordinal);
        uint8_t* d_chunks = nullptr;
        MXD_CUDA(cudaMallocAsync(&d_chunks, nchunks * 32, d->compute));   // cudaMalloc/cudaFree are synchronous and slow
        int rc = enqueue_tree_chunks(c, t, static_cast<const uint8_t*>(piece), nbytes, d_chunks, d->compute);
        if (rc == MXD_OK) {
            cudaError_t e = cudaMemcpyAsync(out, d_chunks, nchunks * 32, cudaMemcpyDeviceToHost, d->compute);
            if (e == cudaSuccess) e = cudaStreamSynchronize(d->compute);
            if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, cudaGetErrorString(e));
            c->d2h += nchunks * 32;
        }
        cudaFreeAsync(d_chunks, d->compute);
        return rc;
    }
    Source src; src.mem = static_cast<const uint8_t*>(piece); src.pinned = (kind == MemKind::Pinned);
    return host_tree_chunks_all(c, cs, t, src, nbytes, out);
}

int mxd_tree_finish(mxd_ctx* h, const uint8_t* chunk_digests, uint64_t nchunks, uint64_t size, const mxd_tree_params* tp,
                    uint8_t root[32]) {
    Tree t;
    if (!handle_ok(h) || !tree_resolve(tp, &t) || !chunk_digests || !root || nchunks == 0) return fail(MXD_ERR_INVALID, "tree_finish: bad arguments");
    const uint64_t expect = size ? (size + t.chunk - 1) / t.chunk : 1;
    if (expect != nchunks) return fail(MXD_ERR_INVALID, "tree_finish: nchunks does not match size/chunk");
    return host_tree_finish(h->core, h->core->devs[0], t, chunk_digests, nchunks, size, root);
}

int mxd_tree_digest(mxd_ctx* h, const void* data, uint64_t size, const mxd_tree_params* tp, uint8_t* chunk_digests,
                    uint64_t* nchunks_out, uint8_t root[32]) {
    Tree t;
    if (!handle_ok(h) || !tree_resolve(tp, &t) || !root || (size && !data)) return fail(MXD_ERR_INVALID, "tree_digest: bad arguments");
    const uint64_t nchunks = size ? (size + t.chunk - 1) / t.chunk : 1;
    std::vector<uint8_t> tmp;
    uint8_t* chunks = chunk_digests;
    if (!chunks) { tmp.resize(nchunks * 32); chunks = tmp.data(); }
    int rc = mxd_tree_chunks(h, data, size, tp, chunks);
    if (rc != MXD_OK) return rc;
    if (nchunks_out) *nchunks_out = nchunks;
    return host_tree_finish(h->core, h->core->devs[0], t, chunks, nchunks, size, root);
}

int mxd_tree_digest_file(mxd_ctx* h, const char* path, const mxd_tree_params* tp, uint8_t* chunk_digests,
                         uint64_t cap_chunks, uint64_t* nchunks_out, uint64_t* size_out, uint8_t root[32]) {
    return mxd_tree_digest_file_tee(h, path, tp, chunk_digests, cap_chunks, nchunks_out, size_out, root, nullptr, nullptr);
}

int mxd_tree_digest_file_tee(mxd_ctx* h, const char* path, const mxd_tree_params* tp, uint8_t* chunk_digests,
                             uint64_t cap_chunks, uint64_t* nchunks_out, uint64_t* size_out, uint8_t root[32],
                             mxd_sink_fn sink, void* user) {
    Tree t;
    if (!handle_ok(h) || !path || !tree_resolve(tp, &t) || !root) return fail(MXD_ERR_INVALID, "tree_digest_file: bad arguments");
    const CancelScope cs(h);
    if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
    int fd = open(path, O_RDONLY | O_CLOEXEC);
    if (fd < 0) return fail(MXD_ERR_IO, std::string("open ") + path + ": " + strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) { int e = errno; close(fd); errno = e; return fail(MXD_ERR_IO, std::string("fstat: ") + strerror(e)); }
    if (S_ISDIR(st.st_mode)) { close(fd); return fail(MXD_ERR_IO, std::string("read ") + path + ": is a directory"); }
    const uint64_t size = (uint64_t)st.st_size;
    const uint64_t nchunks = size ? (size + t.chunk - 1) / t.chunk : 1;
    if (size_out) *size_out = size;
    if (nchunks_out) *nchunks_out = nchunks;
    if (chunk_digests && cap_chunks < nchunks) { close(fd); return fail(MXD_ERR_INVALID, "tree_digest_file: chunk_digests too small"); }
    std::vector<uint8_t> tmp;
    uint8_t* chunks = chunk_digests;
    if (!chunks) { tmp.resize(nchunks * 32); chunks = tmp.data(); }
    Source src; src.fd = fd; src.sink = sink; src.sink_user = user;
    int rc = host_tree_chunks_all(h->core, cs, t, src, size, chunks);
    close(fd);
    if (rc != MXD_OK) return rc;
    return host_tree_finish(h->core, h->core->devs[0], t, chunks, nchunks, size, root);
}

int mxd_tree_load_file(mxd_ctx* h, int dev, const char* path, const mxd_span* dst, uint64_t n, const mxd_tree_params* tp,
                       uint8_t* chunk_digests, uint64_t cap_chunks, uint64_t* nchunks_out, uint64_t* size_out, uint8_t root[32]) {
    Tree t;
    if (!DEV_ARGS_OK(h, dev) || !path || !root || !tree_resolve(tp, &t) || (n && !dst))
        return fail(MXD_ERR_INVALID, "tree_load_file: bad arguments");
    Core* c = h->core;
    DevState* d = c->devs[dev];
    // the destination table: non-empty spans in order, each with its offset in the concatenation
    std::vector<mxd::DevExtent> table;
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uintptr_t p = reinterpret_cast<uintptr_t>(dst[i].ptr);
        const uint64_t len = dst[i].len;
        if (len == 0) continue;
        const std::string which = "tree_load_file: destination " + std::to_string(i);
        if (!p) return fail(MXD_ERR_INVALID, which + " is NULL with a nonzero length");
        if (len > ~0ull - total) return fail(MXD_ERR_INVALID, "tree_load_file: total length overflows 64 bits");
        if (len - 1 > UINTPTR_MAX - p) return fail(MXD_ERR_INVALID, which + " runs past the end of the address space");
        int first_ord = -1, last_ord = -1;
        if (classify(dst[i].ptr, &first_ord) != MemKind::Device || first_ord != d->ordinal ||
            classify(reinterpret_cast<const void*>(p + len - 1), &last_ord) != MemKind::Device || last_ord != d->ordinal)
            return fail(MXD_ERR_INVALID, which + " is not device memory of device " + std::to_string(d->ordinal));
        table.push_back({dst[i].ptr, len, total});
        total += len;
    }
    // the spans are written, so no two may share a byte
    std::vector<const mxd::DevExtent*> by_addr;
    for (const auto& x : table) by_addr.push_back(&x);
    std::sort(by_addr.begin(), by_addr.end(), [](const mxd::DevExtent* a, const mxd::DevExtent* b) { return a->ptr < b->ptr; });
    for (size_t i = 1; i < by_addr.size(); ++i)
        if (static_cast<const uint8_t*>(by_addr[i - 1]->ptr) + by_addr[i - 1]->len > static_cast<const uint8_t*>(by_addr[i]->ptr))
            return fail(MXD_ERR_INVALID, "tree_load_file: destinations overlap");
    const CancelScope cs(h);
    if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
    int fd = open(path, O_RDONLY | O_CLOEXEC);
    if (fd < 0) return fail(MXD_ERR_IO, std::string("open ") + path + ": " + strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) { int e = errno; close(fd); return fail(MXD_ERR_IO, std::string("fstat: ") + strerror(e)); }
    if (S_ISDIR(st.st_mode)) { close(fd); return fail(MXD_ERR_IO, std::string("read ") + path + ": is a directory"); }
    const uint64_t size = (uint64_t)st.st_size;
    if (size != total) {
        close(fd);
        return fail(MXD_ERR_INVALID, "tree_load_file: destinations hold " + std::to_string(total) + " bytes, the file has " + std::to_string(size));
    }
    const uint64_t nchunks = size ? (size + t.chunk - 1) / t.chunk : 1;
    if (chunk_digests && cap_chunks < nchunks) { close(fd); return fail(MXD_ERR_INVALID, "tree_load_file: chunk_digests too small"); }
    const uint64_t n0 = size ? (size + t.leaf - 1) / t.leaf : 1;

    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard guard(d->ordinal);
    Source src; src.fd = fd;
    FileMapGuard fm; fm.attach(&src, size);             // unmapped after the final synchronisation
    cudaStream_t cst = d->compute;
    mxd::DevExtent* d_table = nullptr;
    uint8_t *ws = nullptr, *d_out = nullptr;            // leaf digests; [chunk digests][root]
    std::vector<uint8_t> h_out(nchunks * 32 + 32);
    cudaError_t e = cudaMallocAsync(&ws, n0 * 32, cst);
    if (e == cudaSuccess) e = cudaMallocAsync(&d_out, nchunks * 32 + 32, cst);
    if (e == cudaSuccess && !table.empty()) {
        e = cudaMallocAsync(&d_table, table.size() * sizeof(mxd::DevExtent), cst);
        // from pageable memory: returns once `table` has been staged
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(mxd::DevExtent), cudaMemcpyHostToDevice, cst);
    }
    int rc = (e == cudaSuccess) ? MXD_OK : fail(MXD_ERR_CUDA, std::string("tree_load_file: ") + cudaGetErrorString(e));
    if (rc == MXD_OK) rc = load_leaves(c, cs, d, t, src, size, table, d_table, ws);
    if (rc == MXD_OK) rc = enqueue_levels_to_chunks(c, t, 0, ws, n0, d_out, cst);
    if (rc == MXD_OK) rc = enqueue_tree_finish(c, t, d_out, nchunks, size, d_out + nchunks * 32, cst);
    if (rc == MXD_OK) {
        e = cudaMemcpyAsync(h_out.data(), d_out, nchunks * 32 + 32, cudaMemcpyDeviceToHost, cst);
        if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, std::string("tree_load_file: ") + cudaGetErrorString(e));
    }
    // nothing may still be writing the destinations or reading the file mapping when the call returns
    const cudaError_t e_copy = cudaStreamSynchronize(d->copy);
    const cudaError_t e_comp = cudaStreamSynchronize(cst);
    if (rc == MXD_OK && (e_copy != cudaSuccess || e_comp != cudaSuccess))
        rc = fail(MXD_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e_copy != cudaSuccess ? e_copy : e_comp));
    if (d_table) cudaFreeAsync(d_table, cst);
    if (ws) cudaFreeAsync(ws, cst);
    if (d_out) cudaFreeAsync(d_out, cst);
    close(fd);
    if (rc != MXD_OK) return rc;
    c->d2h += nchunks * 32 + 32;
    if (chunk_digests) memcpy(chunk_digests, h_out.data(), nchunks * 32);
    memcpy(root, h_out.data() + nchunks * 32, 32);
    if (nchunks_out) *nchunks_out = nchunks;
    if (size_out) *size_out = size;
    return MXD_OK;
}

int mxd_tree_chunks_file(mxd_ctx* h, const char* path, uint64_t offset, uint64_t nbytes, const mxd_tree_params* tp, uint8_t* out) {
    Tree t;
    if (!handle_ok(h) || !path || !tree_resolve(tp, &t) || !out) return fail(MXD_ERR_INVALID, "tree_chunks_file: bad arguments");
    if (offset % t.chunk) return fail(MXD_ERR_INVALID, "tree_chunks_file: the piece must start on a chunk boundary");
    const CancelScope cs(h);
    if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
    int fd = open(path, O_RDONLY | O_CLOEXEC);
    if (fd < 0) return fail(MXD_ERR_IO, std::string("open ") + path + ": " + strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) { int e = errno; close(fd); errno = e; return fail(MXD_ERR_IO, std::string("fstat: ") + strerror(e)); }
    if (offset > (uint64_t)st.st_size || nbytes > (uint64_t)st.st_size - offset) { close(fd); return fail(MXD_ERR_IO, "tree_chunks_file: the piece lies outside the file"); }
    Source src; src.fd = fd; src.base = offset;
    int rc = host_tree_chunks_all(h->core, cs, t, src, nbytes, out);
    close(fd);
    return rc;
}

int mxd_tree_digest_files(mxd_ctx* h, const char* const* paths, uint64_t n, const mxd_tree_params* tp, uint8_t* roots,
                          uint64_t* sizes, int* status) {
    Tree t;
    if (!handle_ok(h) || !tree_resolve(tp, &t) || (n && (!paths || !roots))) return fail(MXD_ERR_INVALID, "tree_digest_files: bad arguments");
    if (n == 0) return MXD_OK;
    Core* c = h->core;
    const CancelScope cs(h);
    if (cs.canceled()) return fail(MXD_ERR_CANCELED, "canceled");
    std::vector<TreeFileItem> items(n);
    for (uint64_t i = 0; i < n; ++i) { if (!paths[i]) return fail(MXD_ERR_INVALID, "tree_digest_files: null path"); items[i].path = paths[i]; items[i].root = roots + 32 * i; }
    // files dealt round-robin over the context's devices, one thread per device
    const size_t G = std::min<size_t>(c->devs.size(), n);
    std::vector<std::vector<TreeFileItem*>> share(G);
    for (uint64_t i = 0; i < n; ++i) share[i % G].push_back(&items[i]);
    std::vector<int> rcs(G, MXD_OK); std::vector<std::string> errs(G);
    auto work = [&](size_t g) { rcs[g] = tree_files_on_device(c, cs, c->devs[g], t, share[g]); if (rcs[g] != MXD_OK) errs[g] = last_error(); };
    if (G == 1) work(0);
    else { std::vector<std::thread> th; for (size_t g = 0; g < G; ++g) th.emplace_back(work, g); for (auto& x : th) x.join(); }
    for (size_t g = 0; g < G; ++g) if (rcs[g] != MXD_OK) return fail(rcs[g], errs[g]);
    int first = MXD_OK; std::string first_err;
    for (uint64_t i = 0; i < n; ++i) {
        if (sizes) sizes[i] = items[i].size;
        if (status) status[i] = items[i].status;
        if (items[i].status != MXD_OK && first == MXD_OK) { first = items[i].status; first_err = items[i].error; }
    }
    return first == MXD_OK ? MXD_OK : fail(first, first_err);
}

// ---- whole-message digests ---------------------------------------------------------------------------
// device-resident spans: one launch, no staging; optionally compared with `want` on the device (k_compare)
static int dev_spans_digest(mxd_ctx* h, int first_ord, const mxd_span* spans, uint64_t n, uint8_t* out, const uint8_t* want, uint8_t* ok) {
    Core* c = h->core;
    const int di = dev_index_of(c, first_ord);
    if (di < 0) return fail(MXD_ERR_INVALID, "sha256_batch: data lives on a device this context does not drive");
    DevState* d = c->devs[di];
    DeviceGuard guard(d->ordinal);
    cudaStream_t st = d->compute;
    std::lock_guard<std::mutex> lk(d->mu);
    uint8_t* d_buf = nullptr;   // [spans][digests][want][ok]
    const uint64_t o_dig = n * sizeof(mxd_span), o_want = o_dig + n * 32, o_ok = o_want + n * 32;
    MXD_CUDA(cudaMallocAsync(&d_buf, o_ok + n, st));
    int rc = MXD_OK;
    uint64_t total = 0; for (uint64_t i = 0; i < n; ++i) total += spans[i].len;
    cudaError_t e = cudaMemcpyAsync(d_buf, spans, n * sizeof(mxd_span), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        mxd::MsgJob j{};
        j.spans = d_buf; j.nmsg = n; j.out = d_buf + o_dig; j.finalize = 1; j.one = 1;
        e = mxd::launch_sha256(j, st);
        c->launches++; c->bytes_hashed += total;
    }
    if (e == cudaSuccess && want) {
        e = cudaMemcpyAsync(d_buf + o_want, want, n * 32, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = mxd::launch_compare(d_buf + o_dig, d_buf + o_want, n, d_buf + o_ok, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ok, d_buf + o_ok, n, cudaMemcpyDeviceToHost, st);
        c->launches++; c->d2h += n;
    }
    if (e == cudaSuccess && out) { e = cudaMemcpyAsync(out, d_buf + o_dig, n * 32, cudaMemcpyDeviceToHost, st); c->d2h += n * 32; }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = fail(MXD_ERR_CUDA, cudaGetErrorString(e));
    cudaFreeAsync(d_buf, st);
    return rc;
}

// classify a span list: all host, or all on one device
static int spans_kind(const mxd_span* spans, uint64_t n, bool* on_device, int* ord_out) {
    int ord = -1, first_ord = -1;
    bool all_dev = true, any_dev = false;
    for (uint64_t i = 0; i < n; ++i) {
        if (spans[i].len && !spans[i].ptr) return fail(MXD_ERR_INVALID, "sha256_batch: null span with non-zero length");
        if (spans[i].len == 0) continue;
        if (classify(spans[i].ptr, &ord) == MemKind::Device) {
            any_dev = true;
            if (first_ord < 0) first_ord = ord; else if (ord != first_ord) return fail(MXD_ERR_INVALID, "sha256_batch: spans on different devices");
        } else all_dev = false;
    }
    if (any_dev && !all_dev) return fail(MXD_ERR_INVALID, "sha256_batch: mixing host and device spans");
    *on_device = any_dev; *ord_out = first_ord;
    return MXD_OK;
}

static int first_bad(const std::vector<StreamReq>& reqs, int rc) {
    if (rc != MXD_OK) return rc;
    for (auto& r : reqs) if (r.status != MXD_OK) return fail(r.status, r.error);
    return MXD_OK;
}

int mxd_sha256_batch(mxd_ctx* h, const mxd_span* spans, uint64_t n, uint8_t* out) {
    if (!handle_ok(h) || (n && (!spans || !out))) return fail(MXD_ERR_INVALID, "sha256_batch: bad arguments");
    if (n == 0) return MXD_OK;
    bool on_dev = false; int ord = -1;
    int rc = spans_kind(spans, n, &on_dev, &ord);
    if (rc != MXD_OK) return rc;
    if (on_dev) return dev_spans_digest(h, ord, spans, n, out, nullptr, nullptr);
    std::vector<StreamReq> reqs(n);
    for (uint64_t i = 0; i < n; ++i) { reqs[i].mem = static_cast<const uint8_t*>(spans[i].ptr); reqs[i].size = spans[i].len; reqs[i].whole_out = out + 32 * i; }
    return first_bad(reqs, svc_run(h, reqs));
}

int mxd_sha256(mxd_ctx* h, const void* data, uint64_t n, uint8_t out[32]) {
    if (!handle_ok(h) || !out || (n && !data)) return fail(MXD_ERR_INVALID, "sha256: bad arguments");
    mxd_span sp{data, n};
    return mxd_sha256_batch(h, &sp, 1, out);
}

int mxd_sha256_file_jobs(mxd_ctx* h, mxd_file_job* jobs, uint64_t n) {
    if (!handle_ok(h) || (n && !jobs)) return fail(MXD_ERR_INVALID, "sha256_file_jobs: bad arguments");
    std::vector<StreamReq> reqs(n);
    for (uint64_t i = 0; i < n; ++i) {
        mxd_file_job& jb = jobs[i];
        jb.status = MXD_OK; jb.size = 0;
        if (!jb.path || !jb.out || (jb.nranges && !jb.ranges)) return fail(MXD_ERR_INVALID, "sha256_file_jobs: job " + std::to_string(i) + " has a null path/out/ranges");
        reqs[i].path = jb.path; reqs[i].sink = jb.sink; reqs[i].sink_user = jb.sink_user;
        if (jb.nranges == 0) reqs[i].whole_out = jb.out;
        for (uint64_t k = 0; k < jb.nranges; ++k) {
            if (jb.ranges[k].offset < 0 || jb.ranges[k].length < 0) return fail(MXD_ERR_INVALID, "sha256_file_jobs: negative range");
            reqs[i].ranges.push_back({(uint64_t)jb.ranges[k].offset, (uint64_t)jb.ranges[k].length, jb.out + 32 * k});
        }
    }
    int rc = svc_run(h, reqs);
    for (uint64_t i = 0; i < n; ++i) { jobs[i].status = reqs[i].status; jobs[i].size = reqs[i].size; }
    return first_bad(reqs, rc);
}

int mxd_sha256_files(mxd_ctx* h, const char* const* paths, uint64_t n, uint8_t* out, uint64_t* sizes) {
    if (!handle_ok(h) || (n && (!paths || !out))) return fail(MXD_ERR_INVALID, "sha256_files: bad arguments");
    if (n == 0) return MXD_OK;
    std::vector<mxd_file_job> jobs(n);
    for (uint64_t i = 0; i < n; ++i) { jobs[i] = mxd_file_job{}; jobs[i].path = paths[i]; jobs[i].out = out + 32 * i; }
    int rc = mxd_sha256_file_jobs(h, jobs.data(), n);
    if (sizes) for (uint64_t i = 0; i < n; ++i) sizes[i] = jobs[i].size;
    return rc;
}

int mxd_sha256_file_ranges(mxd_ctx* h, const char* path, const mxd_part* ranges, uint64_t n, uint8_t* out, uint64_t* size,
                           mxd_sink_fn sink, void* user) {
    if (!handle_ok(h) || !path || (n && (!ranges || !out))) return fail(MXD_ERR_INVALID, "sha256_file_ranges: bad arguments");
    if (n == 0 && !sink) return MXD_OK;
    uint8_t dummy[32];
    mxd_file_job jb{};
    jb.path = path; jb.ranges = ranges; jb.nranges = n; jb.out = n ? out : dummy; jb.sink = sink; jb.sink_user = user;
    mxd_part none{0, 0};
    if (n == 0) { jb.ranges = &none; jb.nranges = 1; }     // tee only: hash an empty range
    int rc = mxd_sha256_file_jobs(h, &jb, 1);
    if (size) *size = jb.size;
    return rc;
}

int mxd_sha256_file_parts(mxd_ctx* h, const char* path, const mxd_part* parts, uint64_t n, uint8_t* out) {
    if (!handle_ok(h) || !path || (n && (!parts || !out))) return fail(MXD_ERR_INVALID, "sha256_file_parts: bad arguments");
    if (n == 0) return MXD_OK;
    return mxd_sha256_file_ranges(h, path, parts, n, out, nullptr, nullptr, nullptr);
}

int mxd_sha256_file(mxd_ctx* h, const char* path, uint8_t out[32], uint64_t* size) {
    if (!path) return fail(MXD_ERR_INVALID, "sha256_file: null path");
    const char* paths[1] = {path};
    return mxd_sha256_files(h, paths, 1, out, size);
}

int mxd_verify_batch(mxd_ctx* h, const mxd_span* spans, const uint8_t* want, uint64_t n, uint8_t* ok) {
    if (!handle_ok(h) || (n && (!spans || !want || !ok))) return fail(MXD_ERR_INVALID, "verify_batch: bad arguments");
    if (n == 0) return MXD_OK;
    bool on_dev = false; int ord = -1;
    int rc = spans_kind(spans, n, &on_dev, &ord);
    if (rc != MXD_OK) return rc;
    if (on_dev) return dev_spans_digest(h, ord, spans, n, nullptr, want, ok);   // digests never leave the device
    std::vector<uint8_t> got(n * 32);
    rc = mxd_sha256_batch(h, spans, n, got.data());
    if (rc != MXD_OK) return rc;
    for (uint64_t i = 0; i < n; ++i) ok[i] = memcmp(&got[32 * i], want + 32 * i, 32) == 0;
    return MXD_OK;
}

int mxd_verify_files(mxd_ctx* h, const char* const* paths, const uint8_t* want, uint64_t n, uint8_t* ok) {
    if (!handle_ok(h) || (n && (!paths || !want || !ok))) return fail(MXD_ERR_INVALID, "verify_files: bad arguments");
    std::vector<uint8_t> got(n * 32);
    int rc = mxd_sha256_files(h, paths, n, got.data(), nullptr);
    if (rc != MXD_OK) return rc;
    for (uint64_t i = 0; i < n; ++i) ok[i] = memcmp(&got[32 * i], want + 32 * i, 32) == 0;
    return MXD_OK;
}

// ---- pinned memory -----------------------------------------------------------------------------------
int mxd_host_alloc(mxd_ctx* h, void** out, uint64_t nbytes) {
    if (!handle_ok(h) || !out) return fail(MXD_ERR_INVALID, "host_alloc: bad arguments");
    LocalCpuScope numa(h->core->devs[0]->ordinal);   // place the pages next to the (first) device that will read them
    MXD_CUDA(cudaHostAlloc(out, nbytes, cudaHostAllocPortable));
    return MXD_OK;
}
void mxd_host_free(mxd_ctx*, void* p) { if (p) cudaFreeHost(p); }
int mxd_host_register(mxd_ctx* h, void* p, uint64_t nbytes) {
    if (!handle_ok(h) || !p) return fail(MXD_ERR_INVALID, "host_register: bad arguments");
    MXD_CUDA(cudaHostRegister(p, nbytes, cudaHostRegisterPortable));
    return MXD_OK;
}
int mxd_host_unregister(mxd_ctx* h, void* p) {
    if (!handle_ok(h) || !p) return fail(MXD_ERR_INVALID, "host_unregister: bad arguments");
    MXD_CUDA(cudaHostUnregister(p));
    return MXD_OK;
}

}  // extern "C"
