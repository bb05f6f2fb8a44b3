// C ABI of poseidon252_b200 (include/poseidon252_b200.h): context, host-side sponge bookkeeping
// (io-pattern checks, tag derivation), staging for HOST buffers, kernel launches, fixed-height trees with batched
// updates (p252_mtree_*), sparse fixed-height trees with inserts and removals at any position (p252_smtree_*),
// compact sparse trees stored as sorted present nodes per level (p252_ctree_*),
// variable-length digest batches (p252_hash_batch_varlen), mixed digest batches with a domain, input and output length
// and truncation per item (p252_hash_batch_mixed), and the multi-GPU arity-4 tree build
// (one process per GPU, NCCL all-gather per level).
//
// Mirrors, for the batch path, the reference's public surface (src/lib.rs:13-31):
//   Hash / Domain / io_pattern      src/hash.rs:21-155      -> p252_hash_tag, p252_hash_batch
//   encrypt / decrypt               src/encryption.rs:62-95 -> p252_encrypt_batch, p252_decrypt_batch
//   dhke + encrypt / decrypt        src/encryption.rs:11-43 -> p252_dhke_batch, p252_{en,de}crypt_batch_dhke
//   GENERATOR * r, the sender       src/encryption.rs:22-42 -> p252_fixed_base_batch, p252_encrypt_batch_ephemeral
//   Phoenix stealth addresses (consumer, not the reference) -> p252_stealth_address_batch, p252_stealth_owns_batch
//   jubjub-schnorr sign / verify (consumer, not the reference) -> p252_schnorr_sign_batch, p252_schnorr_verify_batch
//   JubJubAffine::from_bytes / to_bytes (dusk-jubjub, not the reference) -> p252_points_from_bytes, p252_points_to_bytes
//   Phoenix note nullifiers (consumer, not the reference) -> p252_nullifier_batch
//   jubjub-schnorr SignatureDouble, Phoenix note signing (consumer, not the reference) -> p252_schnorr_sign_double_batch,
//     p252_schnorr_verify_double_batch, p252_note_sign_double_batch, p252_schnorr_verify_double_all
//   Phoenix note values (consumer, not the reference) -> p252_value_commit_batch, p252_note_create_batch,
//     p252_note_open_batch
//   JubJub ElGamal, the encrypted sender of a Phoenix note (consumer, not the reference) -> p252_elgamal_encrypt_batch,
//     p252_elgamal_decrypt_batch, p252_note_sender_encrypt_batch, p252_note_sender_decrypt_batch
//   BlsScalar::hash_to_scalar / from_bytes_wide on the device   -> p252_hash_to_scalar_batch,
//     p252_scalars_from_bytes_wide
//   Error                          src/error.rs:11-44      -> p252_status
// No permutation is ever computed on the host: without a CUDA device every batch call fails.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <cub/cub.cuh>
#include <nccl.h>   // types only: the NCCL entry points are resolved at run time (see NcclApi below)

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/poseidon252_b200.h"
#include "host_field.h"
#include "kernels.h"

namespace {

constexpr int kSlots = 3;                    // H2D / compute / D2H overlap for HOST buffers
constexpr size_t kChunkItemsDefault = 1 << 17;   // items per staged chunk (upper bound, also capped by kChunkBytesTarget);
                                                // P252_CHUNK_ITEMS overrides.  e2e ms per 2^20-digest step: 2^15 6.67, 2^16 6.43,
                                                // 2^17 6.43 (equal within run-to-run noise), 157k (bytes cap) 6.48
size_t chunk_items_max() {
    static const size_t v = [] {
        const char* e = getenv("P252_CHUNK_ITEMS");
        const size_t x = e ? (size_t)strtoull(e, nullptr, 10) : kChunkItemsDefault;
        return x >= 1024 ? x : kChunkItemsDefault;
    }();
    return v;
}
constexpr size_t kChunkBytesTarget = 24u << 20;

struct Slot {
    cudaStream_t stream = nullptr;
    void* arena = nullptr;
    size_t arena_bytes = 0;
};

// A device table of per-length tags, tags[len] for len = 0..len (tags[0] = 0) of what `key` names, in a stream-ordered
// allocation, uploaded from a pinned staging buffer whose last upload `ev` marks; staging buffers replaced while their
// upload was still pending wait in `retired` until the context is destroyed.  Rebuilt by tag_table() (below).
struct TagTable {
    p252_fr* dev = nullptr;
    p252_fr* host = nullptr;
    std::vector<p252_fr*> retired;
    size_t host_cap = 0, len = 0;
    uint64_t key = 0;
    cudaEvent_t ev = nullptr;
};

// The device table of p252_fixed_base_batch / p252_encrypt_batch_ephemeral for ONE base, keyed by the base's 64 bytes:
// reused while calls pass that base, rebuilt on the device for another (base_table(), below).
struct BaseTable {
    void* dev = nullptr;
    p252_fr key[2] = {};
};

}  // namespace

struct p252_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    Slot slots[kSlots];
    cudaEvent_t ev_fork = nullptr;
    cudaEvent_t ev_join[kSlots] = {nullptr, nullptr, nullptr};
    uint64_t launches = 0;
    std::string last_error;
    // calls on one context serialise (recursive: public entry points call each other)
    std::recursive_mutex mu;
    // device-side counters (decrypt failures / opening verification / rejected items on DEVICE buffers; slot 0 unless a
    // call counts two things) + their pinned mirror
    static constexpr int kCounters = 2;
    unsigned long long* d_counter = nullptr;
    unsigned long long* h_counter = nullptr;
    size_t coop_max = 0;          // small-batch threshold of the lane-split digest kernel
    // per-length tag tables: p252_hash_batch_varlen (key = domain and out_len) and p252_{en,de}crypt_batch_varlen; two
    // instances, so that alternating digest and encryption calls rebuild neither
    TagTable vt, ct;
    BaseTable bt;   // fixed-base JubJub table
    // the tables of G and G' of the double-key signature and note value calls, only theirs: a wallet that alternates
    // single-base calls with spend signing and note calls keeps all three
    BaseTable bt2[2];
    // test hook: index of the staged chunk that fails in the next host-buffer call (-1 = none)
    long long fail_chunk = -1;
    // multi-GPU
    ncclComm_t comm = nullptr;
    int rank = 0, nranks = 1;
    cudaStream_t comm_stream = nullptr;
    cudaEvent_t ev_level = nullptr, ev_comm = nullptr;
    // per-level timing of the last P252_TIMING tree build
    struct LevelEvents {
        cudaEvent_t k0 = nullptr, k1 = nullptr, g0 = nullptr, g1 = nullptr;
    };
    std::vector<LevelEvents> level_events;
    std::vector<p252_level_timing> level_info;   // static part (nodes, bytes) of the last timed build
    std::vector<char> level_gathered;
    int timed_levels = 0;
    cudaEvent_t ev_tree_end = nullptr;
};

#define P252_LOCK(ctx) std::lock_guard<std::recursive_mutex> lock__((ctx)->mu)

namespace {

// NCCL is bound lazily with dlopen so that (a) single-GPU users carry no NCCL dependency and (b) inside a
// process that already loaded a libnccl.so.2 (e.g. the one bundled with PyTorch) that same copy is used
// instead of a second, possibly older, system copy.
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi& nccl() {
    static NcclApi api;
    if (api.handle) return api;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        api.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD);     // a copy this process already has
        if (api.handle) break;
    }
    for (const char* n : names) {
        if (api.handle) break;
        api.handle = dlopen(n, RTLD_NOW | RTLD_LOCAL);
    }
    if (!api.handle) return api;
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(api.handle, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(api.handle, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(api.handle, "ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(api.handle, "ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(api.handle, "ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
    return api;
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        int cur = -1;
        cudaGetDevice(&cur);
        if (prev >= 0 && cur != prev) cudaSetDevice(prev);
    }
};

int fail_cuda(p252_ctx* ctx, cudaError_t e, const char* where) {
    if (ctx) ctx->last_error = std::string(where) + ": " + cudaGetErrorString(e);
    cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? P252_ERR_OUT_OF_MEMORY : P252_ERR_CUDA;
}
int fail_nccl(p252_ctx* ctx, ncclResult_t e, const char* where) {
    if (ctx) ctx->last_error = std::string(where) + ": " + (nccl().ok ? nccl().GetErrorString(e) : "NCCL unavailable");
    return P252_ERR_NCCL;
}
#define CU(call)                                              \
    do {                                                      \
        cudaError_t e__ = (call);                             \
        if (e__ != cudaSuccess) return fail_cuda(ctx, e__, #call); \
    } while (0)
#define NC(call)                                              \
    do {                                                      \
        ncclResult_t e__ = (call);                            \
        if (e__ != ncclSuccess) return fail_nccl(ctx, e__, #call); \
    } while (0)

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// One staged buffer of a HOST call.
struct Io {
    const void* h_in;    // copied to the device before the launch (may be null)
    void* h_out;         // copied back after the launch (may be null)
    size_t item_bytes;   // bytes per batch item
    bool once = false;   // h_in is ONE item read by every item of the batch: staged once per chunk, never offset
    bool device = false; // h_in / h_out is a device buffer: the launch uses it in place at the chunk's offset, nothing staged
};

// One buffer of a Plan: in a chunk callback, b(d) is its pointer for the chunk, as a T*.
template <typename T>
struct Buf {
    size_t i = 0;
    T* operator()(void* const* d) const { return static_cast<T*>(d[i]); }
};
// The element type of a caller buffer's handle: bytes and integers keep theirs, rows (scalars, points) are untyped.
template <typename T>
using Elem = typename std::conditional<std::is_arithmetic<T>::value, T, void>::type;

// The buffers of a batch call, in the order they are carved from a slot arena and staged, `bytes` per item.  in / out /
// inout are the caller's buffers (used in place when the call's flags say DEVICE); arena buffers are temporaries that
// live in the arena only.  once: one item read by every item of the batch (Io::once).
struct Plan {
    std::vector<Io> ios;
    bool dev;
    explicit Plan(int flags) : dev((flags & P252_MEM_DEVICE) != 0) {}
    template <typename T>
    Buf<Elem<T>> in(const T* p, size_t bytes, bool once = false) { return add<Elem<T>>({p, nullptr, bytes, once, dev}); }
    template <typename T>
    Buf<Elem<T>> out(T* p, size_t bytes) { return add<Elem<T>>({nullptr, p, bytes, false, dev}); }
    template <typename T>
    Buf<Elem<T>> inout(T* p, size_t bytes) { return add<Elem<T>>({p, p, bytes, false, dev}); }
    template <typename T = void>
    Buf<T> arena(size_t bytes, bool once = false) { return add<T>({nullptr, nullptr, bytes, once}); }
    template <typename T>
    Io& operator[](Buf<T> b) { return ios[b.i]; }
  private:
    template <typename T>
    Buf<T> add(Io io) { ios.push_back(io); return {ios.size() - 1}; }
};

int join_slots(p252_ctx* ctx, int rc, bool wipe);

// Every kernel launch of the library goes through here: a failed launch is reported, a successful one counted.
int launched(p252_ctx* ctx, cudaError_t le) {
    if (le != cudaSuccess) return fail_cuda(ctx, le, "kernel launch");
    ctx->launches++;
    return P252_OK;
}
// Enqueue one kernel through launched(); a failed launch returns its status, so no later kernel is enqueued.
#define LAUNCH(call)                                                             \
    do {                                                                         \
        if (const int rc__ = launched(ctx, (call)); rc__ != P252_OK) return rc__; \
    } while (0)

// Tail of every DEVICE-buffer call: the status of its work, then synchronous unless P252_ASYNC.
int device_done(p252_ctx* ctx, int rc, int flags) {
    if (rc != P252_OK) return rc;
    if (!(flags & P252_ASYNC)) CU(cudaStreamSynchronize(ctx->stream));
    return P252_OK;
}

// number of zero bytes of ok[0, n): failures counted on the host
size_t count_zero(const uint8_t* ok, size_t n) {
    size_t bad = 0;
    for (size_t i = 0; i < n; ++i) bad += ok[i] ? 0 : 1;
    return bad;
}

// The layout of a set of device temporaries: 256-byte aligned pieces, taken in order.  Over a null base it only adds up
// the size, so that one layout function both sizes and carves a buffer.
struct Carve {
    uint8_t* base = nullptr;
    size_t used = 0;
    template <typename T>
    T* take(size_t count) {
        T* r = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += (count * sizeof(T) + 255) / 256 * 256;
        return r;
    }
};

// Temporaries of one call: layout(Carve&) places them in one stream-ordered allocation on `st`, body() runs, and the
// allocation is freed in stream order whatever body() returned; the free's error is reported only when body() succeeded.
template <typename Layout, typename Body>
int with_scratch(p252_ctx* ctx, cudaStream_t st, Layout layout, Body body) {
    Carve c;
    layout(c);
    CU(cudaMallocAsync(reinterpret_cast<void**>(&c.base), c.used, st));
    c.used = 0;
    layout(c);
    const int rc = body();
    const cudaError_t fe = cudaFreeAsync(c.base, st);
    if (rc != P252_OK) return rc;
    if (fe != cudaSuccess) return fail_cuda(ctx, fe, "cudaFreeAsync");
    return P252_OK;
}

// Grow a slot's arena to at least `need` bytes.  The old arena is released only after the slot stream has drained, and
// is cleared first when it may hold secrets (wipe).
int slot_reserve(p252_ctx* ctx, Slot& sl, size_t need, bool wipe) {
    if (sl.arena_bytes >= need) return P252_OK;
    CU(cudaStreamSynchronize(sl.stream));
    if (sl.arena) {
        if (wipe) CU(cudaMemset(sl.arena, 0, sl.arena_bytes));
        CU(cudaFree(sl.arena));
    }
    sl.arena = nullptr;
    sl.arena_bytes = 0;
    CU(cudaMalloc(&sl.arena, need));
    sl.arena_bytes = need;
    return P252_OK;
}

// A HOST call on the slot streams: they first wait for everything already enqueued on the context stream, then
// body(fail_at) stages its chunks (fail_at: the chunk p252_debug_fail_chunk makes fail, taken one shot).
// wipe = true: the staging arenas held secrets (shared secret, nonce, plaintext); they are cleared before
// returning (the reference's dependencies zeroize sponge state, Cargo.toml:15,17 "zeroize").
// Whatever body returns, the common exit join_slots runs: slot streams are joined back into the context stream, the
// arenas are wiped if asked, and the call returns only after everything enqueued has finished -- so on an error no copy
// into the caller's buffers is still in flight and no secret is left staged.
template <typename Body>
int on_slots(p252_ctx* ctx, bool wipe, Body body) {
    const long long fail_at = ctx->fail_chunk;
    ctx->fail_chunk = -1;
    auto run = [&]() -> int {
        CU(cudaEventRecord(ctx->ev_fork, ctx->stream));
        for (int s = 0; s < kSlots; ++s) CU(cudaStreamWaitEvent(ctx->slots[s].stream, ctx->ev_fork, 0));
        return body(fail_at);
    };
    return join_slots(ctx, run(), wipe);
}

int injected_fault(p252_ctx* ctx) { return fail_cuda(ctx, cudaErrorLaunchFailure, "kernel launch (injected fault)"); }

// The largest chunk run_host_pipeline stages for `ios` and n > 0 items
size_t pipeline_chunk(const std::vector<Io>& ios, size_t n) {
    size_t per_item = 0;
    for (auto& io : ios)
        if (!io.once && !io.device) per_item += (io.item_bytes + 15) / 16 * 16;
    size_t chunk = std::max<size_t>(1024, std::min(chunk_items_max(), kChunkBytesTarget / std::max<size_t>(per_item, 1)));
    chunk = (chunk + 127) / 128 * 128;
    return chunk > n ? n : chunk;
}

// The chunk loop of both pipelines, on the slot streams (on_slots): chunk k goes to slot k % kSlots, whose arena is
// grown to hold every staged buffer of `ios` and carved into one region per buffer; the chunk's inputs are copied in
// (DEVICE buffers are used in place at the chunk's offset), and then body(d, off, cnt, st) enqueues the chunk's work
// on the slot stream st, d being the chunk's buffers in the order of `ios` (valid until that slot's next chunk).
// Ramp-up (batches of several chunks only): the first chunks are small (chunk/8, /4, /2) so that the first kernel
// starts after a ~1 MiB copy instead of a full chunk's; from the fourth chunk on every chunk has the full size.  A batch
// that fits one chunk is one launch.
template <typename Body>
int stage_chunks(p252_ctx* ctx, const std::vector<Io>& ios, size_t n, bool wipe, Body body) {
    if (n == 0) return P252_OK;
    const size_t chunk = pipeline_chunk(ios, n);
    std::vector<void*> d[kSlots];
    auto carve = [&](void* arena, std::vector<void*>& dd) {
        dd.resize(ios.size());
        Carve c{static_cast<uint8_t*>(arena)};
        for (size_t b = 0; b < ios.size(); ++b)
            if (!ios[b].device) dd[b] = c.take<uint8_t>((ios[b].once ? 1 : chunk) * ios[b].item_bytes);
        return c.used;
    };
    const size_t need = carve(nullptr, d[kSlots - 1]);
    return on_slots(ctx, wipe, [&](long long fail_at) -> int {
        size_t k = 0, cur = (n > 2 * chunk) ? std::max<size_t>(1024, chunk / 8 / 128 * 128) : chunk;
        for (size_t off = 0, cnt = 0; off < n; off += cnt, ++k, cur = std::min(chunk, cur * 2)) {
            cnt = std::min(cur, n - off);
            const int s = (int)(k % kSlots);
            Slot& sl = ctx->slots[s];
            int rc = slot_reserve(ctx, sl, need, wipe);
            if (rc != P252_OK) return rc;
            carve(sl.arena, d[s]);
            for (size_t b = 0; b < ios.size(); ++b) {
                const Io& io = ios[b];
                const size_t at = io.once ? 0 : off * io.item_bytes;
                if (io.device)
                    d[s][b] = io.h_out ? static_cast<uint8_t*>(io.h_out) + at
                                       : const_cast<uint8_t*>(static_cast<const uint8_t*>(io.h_in) + at);
                else if (io.h_in)
                    CU(cudaMemcpyAsync(d[s][b], static_cast<const uint8_t*>(io.h_in) + at,
                                       (io.once ? 1 : cnt) * io.item_bytes, cudaMemcpyHostToDevice, sl.stream));
            }
            if ((long long)k == fail_at) return injected_fault(ctx);
            if ((rc = body(d[s].data(), off, cnt, sl.stream)) != P252_OK) return rc;
        }
        return P252_OK;
    });
}

// The output copies of a staged chunk (d: its buffers, at items [off, off + cnt)) back to the caller's HOST buffers.
int copy_out(p252_ctx* ctx, const std::vector<Io>& ios, void* const* d, size_t off, size_t cnt, cudaStream_t st) {
    for (size_t b = 0; b < ios.size(); ++b)
        if (ios[b].h_out && !ios[b].device)
            CU(cudaMemcpyAsync(static_cast<uint8_t*>(ios[b].h_out) + off * ios[b].item_bytes, d[b], cnt * ios[b].item_bytes,
                               cudaMemcpyDeviceToHost, st));
    return P252_OK;
}

// Fixed-size HOST batches: the items stream through the slot arenas in chunks, each buffer of `ios` staged in its own
// region.  launch(d, cnt, st) enqueues a chunk's kernels, each through launched(), and returns a P252_* status; the
// chunk's output copies follow it on the same slot stream.
template <typename Launch>
int run_host_pipeline(p252_ctx* ctx, const std::vector<Io>& ios, size_t n, Launch launch, bool wipe = false) {
    return stage_chunks(ctx, ios, n, wipe, [&](void** d, size_t off, size_t cnt, cudaStream_t st) {
        const int rc = launch(d, cnt, st);
        return rc != P252_OK ? rc : copy_out(ctx, ios, d, off, cnt, st);
    });
}

// Fixed-size batches whose chunks run in two phases, where the host needs something the first phase computed (a count)
// before it can enqueue the second: the chunks are staged as in run_host_pipeline, but chunk c's second(d, cnt, st) and
// its output copies are enqueued after chunk c + 1's first(d, cnt, st), so that while the host waits for chunk c the
// device already has the next chunk's first phase queued on another slot, and consecutive chunks overlap.  Both callbacks
// enqueue through launched() and return a P252_* status.
template <typename First, typename Second>
int run_host_pipeline2(p252_ctx* ctx, const std::vector<Io>& ios, size_t n, First first, Second second, bool wipe = false) {
    struct Chunk { void** d; size_t off, cnt; cudaStream_t st; } prev{};
    auto finish = [&](const Chunk& c) -> int {
        const int rc = second(c.d, c.cnt, c.st);
        return rc != P252_OK ? rc : copy_out(ctx, ios, c.d, c.off, c.cnt, c.st);
    };
    return stage_chunks(ctx, ios, n, wipe, [&](void** d, size_t off, size_t cnt, cudaStream_t st) -> int {
        int rc = first(d, cnt, st);
        if (rc != P252_OK || (prev.d && (rc = finish(prev)) != P252_OK)) return rc;
        prev = Chunk{d, off, cnt, st};
        return off + cnt == n ? finish(prev) : P252_OK;   // the last chunk
    });
}

// Common exit of every HOST call that ran on the slot streams (success and failure): wipe, join, drain.
int join_slots(p252_ctx* ctx, int rc, bool wipe) {
    const std::string first_error = ctx->last_error;
    cudaError_t ce = cudaSuccess;
    auto keep = [&](cudaError_t e) {
        if (e != cudaSuccess && ce == cudaSuccess) ce = e;
    };
    for (int s = 0; s < kSlots; ++s) {
        Slot& sl = ctx->slots[s];
        if (wipe && sl.arena) keep(cudaMemsetAsync(sl.arena, 0, sl.arena_bytes, sl.stream));
        keep(cudaEventRecord(ctx->ev_join[s], sl.stream));
        keep(cudaStreamWaitEvent(ctx->stream, ctx->ev_join[s], 0));
    }
    keep(cudaStreamSynchronize(ctx->stream));   // HOST calls are synchronous on return, like the reference
    if (rc != P252_OK) {
        // make sure nothing is in flight even if the join itself could not be enqueued
        for (int s = 0; s < kSlots; ++s) cudaStreamSynchronize(ctx->slots[s].stream);
        cudaGetLastError();
        ctx->last_error = first_error;
        return rc;
    }
    if (ce != cudaSuccess) return fail_cuda(ctx, ce, "host pipeline join");
    return P252_OK;
}

// DEVICE-buffer calls that count failures on the device: zero the first `count` counters before the launch ...
int counter_begin(p252_ctx* ctx, int count = 1) {
    CU(cudaMemsetAsync(ctx->d_counter, 0, count * sizeof(unsigned long long), ctx->stream));
    return P252_OK;
}
template <typename T>
void CUDART_CB publish_counter(void* arg) {
    auto* pr = static_cast<std::pair<const unsigned long long*, T*>*>(arg);
    *pr->second = std::is_same<T, uint8_t>::value ? (T)(*pr->first != 0) : (T)*pr->first;
    delete pr;
}
// ... and after it copy counter `slot` to the pinned mirror and from there to the caller's size_t, or as a yes / no answer
// (0 or 1) to the caller's byte (a host function on the stream, so that P252_ASYNC callers see it after p252_sync).
template <typename T>
int counter_end(p252_ctx* ctx, T* out, int slot = 0) {
    if (!out) return P252_OK;
    CU(cudaMemcpyAsync(ctx->h_counter + slot, ctx->d_counter + slot, sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                       ctx->stream));
    auto* pr = new std::pair<const unsigned long long*, T*>(ctx->h_counter + slot, out);
    cudaError_t e = cudaLaunchHostFunc(ctx->stream, publish_counter<T>, pr);
    if (e != cudaSuccess) {
        delete pr;
        return fail_cuda(ctx, e, "cudaLaunchHostFunc");
    }
    return P252_OK;
}

bool one_or_n(size_t k, size_t n) { return k == 1 || k == n; }

// The buffer checks of a fixed-length batch call of n items: with n > 0 no listed buffer may be NULL, and DEVICE buffers
// must be 16-byte aligned (`rows`: field elements, scalars, points) or 8-byte aligned (`idx`: uint64 indices).  Result
// bytes (`bytes`: ok / owned / verified) need no alignment.
bool args_ok(size_t n, int flags, std::initializer_list<const void*> rows, std::initializer_list<const void*> bytes = {},
             std::initializer_list<const void*> idx = {}) {
    const bool dev = (flags & P252_MEM_DEVICE) != 0;
    for (auto list : {rows, bytes, idx})
        for (const void* b : list)
            if (n && !b) return false;
    for (const void* b : rows)
        if (dev && !aligned16(b)) return false;
    for (const void* b : idx)
        if (dev && (reinterpret_cast<uintptr_t>(b) & 7)) return false;
    return true;
}

// The failure counts of a fixed-length batch call, and the tail of its DEVICE calls.  The constructor zeroes the caller's
// counts, begin() zeroes the device counters before the first launch, counter(i) is device counter i for the kernels
// (null where nothing is counted on the device), and end(rc) publishes the counts and returns the call's status.
//   ok-recount (the constructor): HOST calls recount the zero bytes of ok[0, n) on the host, DEVICE calls count on device
//     counter 0.  Without a count pointer only the DEVICE tail is left (device_done).
//   device-counted (Counts::device): both memory spaces count on device counters 0 and 1, for when ok[] alone cannot tell
//     what is counted; counter 1 may instead be a yes / no answer published as one byte.  HOST calls return with them
//     published.
struct Counts {
    p252_ctx* ctx;
    int flags;
    size_t* count[2];
    uint8_t* answer = nullptr;
    const uint8_t* ok;
    size_t n;
    bool device_counted = false;

    Counts(p252_ctx* c, int f, size_t* failed = nullptr, const uint8_t* ok_ = nullptr, size_t n_ = 0)
        : ctx(c), flags(f), count{failed, nullptr}, ok(ok_), n(n_) {
        if (failed) *failed = 0;
    }
    static Counts device(p252_ctx* c, int f, size_t* c0, size_t* c1 = nullptr, uint8_t* answer = nullptr) {
        Counts k(c, f, c0);
        if ((k.count[1] = c1)) *c1 = 0;
        k.answer = answer;
        k.device_counted = true;
        return k;
    }
    bool on_device() const { return device_counted || (flags & P252_MEM_DEVICE); }
    unsigned long long* counter(int i) const {
        return on_device() && (count[i] || (i == 1 && answer)) ? ctx->d_counter + i : nullptr;
    }
    int begin() const {
        if (!counter(0) && !counter(1)) return P252_OK;
        return counter_begin(ctx, counter(1) ? 2 : 1);
    }
    int end(int rc) const {
        if (!on_device()) {
            if (rc == P252_OK && count[0]) *count[0] = count_zero(ok, n);
            return rc;
        }
        if (rc == P252_OK) rc = counter_end(ctx, count[0], 0);
        if (rc == P252_OK) rc = counter_end(ctx, count[1], 1);
        if (rc == P252_OK) rc = counter_end(ctx, answer, 1);
        return device_done(ctx, rc, (flags & P252_MEM_DEVICE) ? flags : 0);   // HOST calls return with their counts published
    }
};

// A single-launch batch call states its launch once, as launch(d, cnt, st) over the buffers of `plan`: DEVICE buffers run
// it once on the context stream with the caller's pointers, HOST buffers through run_host_pipeline with the staged ones.
template <typename Launch>
int launch_batch(const Counts& counts, const Plan& plan, size_t n, Launch launch, bool wipe = false) {
    if (!(counts.flags & P252_MEM_DEVICE)) return counts.end(run_host_pipeline(counts.ctx, plan.ios, n, launch, wipe));
    if (n == 0) return P252_OK;
    const int rc = counts.begin();
    if (rc != P252_OK) return rc;
    std::vector<void*> d;
    for (const Io& io : plan.ios) d.push_back(io.h_out ? io.h_out : const_cast<void*>(io.h_in));
    return counts.end(launch(d.data(), n, counts.ctx->stream));
}

// A batch call that runs through the slot arenas for both memory spaces (DEVICE buffers used in place, chunk by chunk):
// the device counters are zeroed, the chunks run, and the counts are published.  Called after the n == 0 return.
template <typename Launch>
int staged_batch(const Counts& counts, const Plan& plan, size_t n, Launch launch, bool wipe = false) {
    const int rc = counts.begin();
    return counts.end(rc != P252_OK ? rc : run_host_pipeline(counts.ctx, plan.ios, n, launch, wipe));
}

uint64_t domain_sep(int domain, bool* ok) {
    *ok = true;
    switch (domain) {
        case P252_DOMAIN_MERKLE4: return 0x000000000000000fULL;      // src/hash.rs:47
        case P252_DOMAIN_MERKLE2: return 0x0000000000000003ULL;      // src/hash.rs:49
        case P252_DOMAIN_ENCRYPTION: return 0x0000000100000000ULL;   // src/hash.rs:51
        case P252_DOMAIN_OTHER: return 0;                            // src/hash.rs:53
    }
    *ok = false;
    return 0;
}

const uint64_t* limbs(const p252_fr* f) { return f->l; }

// HOST openings in the format of k_merkle_open (kernels.h): for leaf idx[i] and level l < depth the sibling group of level
// l, slots at or beyond lv.m[l] read as zero.  The indices are validated by the caller.
void open_host(const p252_fr* leaves, const p252_fr* nodes, const uint64_t* idx, size_t n, int arity, int depth,
               const p252::OpenLevels& lv, p252_fr* paths) {
    const uint64_t A = (uint64_t)arity;
    for (size_t i = 0; i < n; ++i) {
        uint64_t j = idx[i];
        for (int l = 0; l < depth; ++l) {
            const uint64_t group = j / A;
            const p252_fr* src = (l == 0 ? leaves : nodes + lv.off[l]) + group * A;
            p252_fr* dst = paths + (i * (size_t)depth + (size_t)l) * A;
            for (uint64_t q = 0; q < A; ++q) {
                if (group * A + q < lv.m[l])
                    dst[q] = src[q];
                else
                    memset(&dst[q], 0, sizeof(p252_fr));
            }
            j = group;
        }
    }
}

}  // namespace

extern "C" {

const char* p252_version(void) { return "poseidon252_b200 0.1.0 (sm_90a)"; }

const char* p252_strerror(int status) {
    switch (status) {
        case P252_OK: return "ok";
        case P252_ERR_IO_PATTERN_VIOLATION: return "IOPatternViolation";
        case P252_ERR_INVALID_IO_PATTERN: return "InvalidIOPattern";
        case P252_ERR_TOO_FEW_INPUT_ELEMENTS: return "TooFewInputElements";
        case P252_ERR_ENCRYPTION_FAILED: return "EncryptionFailed";
        case P252_ERR_DECRYPTION_FAILED: return "DecryptionFailed";
        case P252_ERR_INVALID_POINT: return "InvalidPoint";
        case P252_ERR_INVALID_ARGUMENT: return "invalid argument";
        case P252_ERR_CUDA: return "CUDA error";
        case P252_ERR_NCCL: return "NCCL error";
        case P252_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (there is no CPU fallback)";
        case P252_ERR_OUT_OF_MEMORY: return "out of device memory";
    }
    return "unknown status";
}

int p252_device_count(int* count) {
    if (!count) return P252_ERR_INVALID_ARGUMENT;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    *count = n;
    return P252_OK;
}

int p252_create_on_stream(int device, void* cuda_stream, p252_ctx** out) {
    if (!out) return P252_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        return P252_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n) return P252_ERR_INVALID_ARGUMENT;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return P252_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return P252_ERR_NO_DEVICE;   // kernels are sm_90a SASS only
    p252_ctx* ctx = new p252_ctx();
    ctx->device = device;
    ctx->coop_max = p252::coop_max_items(prop.multiProcessorCount);
    DeviceGuard g(device);
    auto bail = [&](cudaError_t e, const char* w) {
        int rc = fail_cuda(nullptr, e, w);
        p252_destroy(ctx);
        return rc;
    };
    cudaError_t e;
    if (cuda_stream) {
        ctx->stream = static_cast<cudaStream_t>(cuda_stream);
        ctx->own_stream = false;
    } else {
        if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess)
            return bail(e, "cudaStreamCreate");
        ctx->own_stream = true;
    }
    for (int s = 0; s < kSlots; ++s) {
        if ((e = cudaStreamCreateWithFlags(&ctx->slots[s].stream, cudaStreamNonBlocking)) != cudaSuccess)
            return bail(e, "cudaStreamCreate");
        if ((e = cudaEventCreateWithFlags(&ctx->ev_join[s], cudaEventDisableTiming)) != cudaSuccess)
            return bail(e, "cudaEventCreate");
    }
    if ((e = cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming)) != cudaSuccess)
        return bail(e, "cudaEventCreate");
    if ((e = cudaEventCreateWithFlags(&ctx->ev_level, cudaEventDisableTiming)) != cudaSuccess)
        return bail(e, "cudaEventCreate");
    if ((e = cudaEventCreateWithFlags(&ctx->ev_comm, cudaEventDisableTiming)) != cudaSuccess)
        return bail(e, "cudaEventCreate");
    if ((e = cudaEventCreate(&ctx->ev_tree_end)) != cudaSuccess) return bail(e, "cudaEventCreate");
    for (TagTable* t : {&ctx->vt, &ctx->ct})
        if ((e = cudaEventCreateWithFlags(&t->ev, cudaEventDisableTiming)) != cudaSuccess) return bail(e, "cudaEventCreate");
    const size_t counter_bytes = p252_ctx::kCounters * sizeof(unsigned long long);
    if ((e = cudaMalloc(reinterpret_cast<void**>(&ctx->d_counter), counter_bytes)) != cudaSuccess)
        return bail(e, "cudaMalloc");
    if ((e = cudaHostAlloc(reinterpret_cast<void**>(&ctx->h_counter), counter_bytes, cudaHostAllocPortable)) != cudaSuccess)
        return bail(e, "cudaHostAlloc");
    memset(ctx->h_counter, 0, counter_bytes);
    *out = ctx;
    return P252_OK;
}

int p252_create(int device, p252_ctx** out) { return p252_create_on_stream(device, nullptr, out); }

void p252_destroy(p252_ctx* ctx) {
    if (!ctx) return;
    DeviceGuard g(ctx->device);
    if (ctx->comm && nccl().ok) nccl().CommDestroy(ctx->comm);
    if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
    for (int s = 0; s < kSlots; ++s) {
        if (ctx->slots[s].stream) {
            cudaStreamSynchronize(ctx->slots[s].stream);
            cudaStreamDestroy(ctx->slots[s].stream);
        }
        if (ctx->slots[s].arena) cudaFree(ctx->slots[s].arena);
        if (ctx->ev_join[s]) cudaEventDestroy(ctx->ev_join[s]);
    }
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_level) cudaEventDestroy(ctx->ev_level);
    if (ctx->ev_comm) cudaEventDestroy(ctx->ev_comm);
    if (ctx->ev_tree_end) cudaEventDestroy(ctx->ev_tree_end);
    for (auto& le : ctx->level_events)
        for (cudaEvent_t ev : {le.k0, le.k1, le.g0, le.g1})
            if (ev) cudaEventDestroy(ev);
    for (TagTable* t : {&ctx->vt, &ctx->ct})
        if (t->dev) cudaFreeAsync(t->dev, ctx->stream);
    for (BaseTable* t : {&ctx->bt, &ctx->bt2[0], &ctx->bt2[1]})
        if (t->dev) cudaFreeAsync(t->dev, ctx->stream);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);   // pending host functions reference h_counter
    for (TagTable* t : {&ctx->vt, &ctx->ct}) {
        if (t->host) cudaFreeHost(t->host);
        for (p252_fr* h : t->retired) cudaFreeHost(h);
        if (t->ev) cudaEventDestroy(t->ev);
    }
    if (ctx->d_counter) cudaFree(ctx->d_counter);
    if (ctx->h_counter) cudaFreeHost(ctx->h_counter);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int p252_sync(p252_ctx* ctx) {
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    CU(cudaStreamSynchronize(ctx->stream));
    return P252_OK;
}

int p252_get_kernel_info(p252_kernel_info* out) {
    if (!out || out->struct_size < sizeof(p252_kernel_info)) return P252_ERR_INVALID_ARGUMENT;
    int t = 0, b = 0;
    p252::kernel_launch_shape(&t, &b);
    out->struct_size = (uint32_t)sizeof(p252_kernel_info);
    out->wide_mul_per_permutation = p252::wide_mul_per_permutation();
    out->dfma_per_permutation = p252::dfma_per_permutation();
    out->montmul_per_permutation = 365;
    out->threads_per_block = (uint32_t)t;
    out->min_blocks_per_sm = (uint32_t)b;
    return P252_OK;
}

int p252_set_small_batch_max(p252_ctx* ctx, size_t max_items) {
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    ctx->coop_max = max_items;
    return P252_OK;
}

int p252_debug_fail_chunk(p252_ctx* ctx, long long k) {
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    ctx->fail_chunk = k;
    return P252_OK;
}

int p252_debug_staging_nonzero(p252_ctx* ctx, size_t* nonzero_bytes) {
    if (!ctx || !nonzero_bytes) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    size_t bad = 0;
    for (int s = 0; s < kSlots; ++s) {
        Slot& sl = ctx->slots[s];
        if (!sl.arena) continue;
        CU(cudaStreamSynchronize(sl.stream));
        std::vector<uint8_t> h(sl.arena_bytes);
        CU(cudaMemcpy(h.data(), sl.arena, sl.arena_bytes, cudaMemcpyDeviceToHost));
        for (uint8_t v : h) bad += v ? 1 : 0;
    }
    *nonzero_bytes = bad;
    return P252_OK;
}

const char* p252_last_error(const p252_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }
uint64_t p252_launch_count(const p252_ctx* ctx) { return ctx ? ctx->launches : 0; }

int p252_host_alloc(size_t bytes, void** out) {
    if (!out) return P252_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    p252_ctx* ctx = nullptr;
    CU(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable));
    return P252_OK;
}
int p252_host_free(void* p) {
    p252_ctx* ctx = nullptr;
    if (p) CU(cudaFreeHost(p));
    return P252_OK;
}

// ---- host-side sponge bookkeeping ---------------------------------------------------------------
int p252_domain_separator(int domain, uint64_t* out) {
    bool ok;
    uint64_t v = domain_sep(domain, &ok);
    if (!ok || !out) return P252_ERR_INVALID_ARGUMENT;
    *out = v;
    return P252_OK;
}

int p252_tag_input(const uint32_t* calls, size_t ncalls, uint64_t dsep, uint8_t* out, size_t* out_len) {
    if (!calls || !out_len) return P252_ERR_INVALID_ARGUMENT;
    // a valid io-pattern starts with an absorb, ends with a squeeze and has no zero-length call
    if (ncalls == 0 || !(calls[0] & 0x80000000u) || (calls[ncalls - 1] & 0x80000000u)) return P252_ERR_INVALID_IO_PATTERN;
    std::vector<uint32_t> words;
    for (size_t i = 0; i < ncalls; ++i) {
        if ((calls[i] & 0x7fffffffu) == 0) return P252_ERR_INVALID_IO_PATTERN;
        if (!words.empty() && ((words.back() ^ calls[i]) & 0x80000000u) == 0)
            words.back() += calls[i] & 0x7fffffffu;   // aggregate consecutive calls of one kind
        else
            words.push_back(calls[i]);
    }
    const size_t need = words.size() * 4 + 8;
    if (!out || *out_len < need) {
        *out_len = need;
        return out ? P252_ERR_INVALID_ARGUMENT : P252_OK;
    }
    size_t p = 0;
    for (uint32_t w : words)
        for (int s = 24; s >= 0; s -= 8) out[p++] = (uint8_t)(w >> s);
    for (int s = 56; s >= 0; s -= 8) out[p++] = (uint8_t)(dsep >> s);
    *out_len = need;
    return P252_OK;
}

int p252_hash_to_scalar(const uint8_t* bytes, size_t len, p252_fr* out) {
    if (!out || (!bytes && len)) return P252_ERR_INVALID_ARGUMENT;
    uint8_t digest[64];
    p252::host::blake2b512(bytes, len, digest);
    p252::host::from_bytes_wide(out->l, digest);
    return P252_OK;
}

int p252_tag(const uint32_t* calls, size_t ncalls, uint64_t dsep, p252_fr* tag) {
    if (!tag) return P252_ERR_INVALID_ARGUMENT;
    std::vector<uint8_t> buf(ncalls * 4 + 8 + 8);
    size_t len = buf.size();
    int rc = p252_tag_input(calls, ncalls, dsep, buf.data(), &len);
    if (rc != P252_OK) return rc;
    return p252_hash_to_scalar(buf.data(), len, tag);
}

int p252_hash_tag(int domain, size_t in_len, size_t out_len, p252_fr* tag) {
    bool ok;
    const uint64_t dsep = domain_sep(domain, &ok);
    if (!ok || !tag) return P252_ERR_INVALID_ARGUMENT;
    // io_pattern, src/hash.rs:62-85
    if (domain == P252_DOMAIN_MERKLE2 && (in_len != 2 || out_len != 1)) return P252_ERR_IO_PATTERN_VIOLATION;
    if (domain == P252_DOMAIN_MERKLE4 && (in_len != 4 || out_len != 1)) return P252_ERR_IO_PATTERN_VIOLATION;
    if (in_len == 0 || out_len == 0) return P252_ERR_INVALID_IO_PATTERN;
    if (in_len >= 0x80000000ull || out_len >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    const uint32_t calls[2] = {0x80000000u | (uint32_t)in_len, (uint32_t)out_len};
    return p252_tag(calls, 2, dsep, tag);
}

int p252_encryption_tag(size_t L, p252_fr* tag) {
    if (!tag) return P252_ERR_INVALID_ARGUMENT;
    if (L == 0) return P252_ERR_INVALID_IO_PATTERN;
    if (L >= 0x7ffffff0ull) return P252_ERR_INVALID_ARGUMENT;
    // [Absorb(2), Absorb(1), Squeeze(L), Absorb(L), Squeeze(1)], src/encryption.rs:67-73
    const uint32_t calls[5] = {0x80000002u, 0x80000001u, (uint32_t)L, 0x80000000u | (uint32_t)L, 1u};
    bool ok;
    return p252_tag(calls, 5, domain_sep(P252_DOMAIN_ENCRYPTION, &ok), tag);
}

// ---- batch entry points ---------------------------------------------------------------------------
static int permute_impl(p252_ctx* ctx, p252_fr* states, size_t n, int flags, bool dense) {
    if (!ctx || !args_ok(n, flags, {states})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    Plan p(flags);
    const auto d_states = p.inout(states, 160);
    return launch_batch(Counts(ctx, flags), p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_permute(d_states(d), cnt, dense, ctx->coop_max, st));
    });
}

int p252_permute_batch(p252_ctx* ctx, p252_fr* states, size_t n, int flags) {
    return permute_impl(ctx, states, n, flags, false);
}
int p252_permute_batch_dense(p252_ctx* ctx, p252_fr* states, size_t n, int flags) {
    return permute_impl(ctx, states, n, flags, true);
}

// Here and in the encrypt / decrypt batches a NULL buffer is refused before the io pattern is checked, a misaligned
// DEVICE buffer (args_ok) after it.
static int digest_impl(p252_ctx* ctx, const p252_fr* tag, const p252_fr* in, size_t n, size_t in_len, p252_fr* out,
                       size_t out_len, int flags, bool truncate) {
    if (!ctx || !tag || ((!in || !out) && n)) return P252_ERR_INVALID_ARGUMENT;
    if (in_len == 0 || out_len == 0) return P252_ERR_INVALID_IO_PATTERN;
    if (in_len > 0x7fffffffull / 32 || out_len > 0x7fffffffull / 32 || !args_ok(n, flags, {in, out}))
        return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const uint32_t il = (uint32_t)in_len, ol = (uint32_t)out_len;
    Plan p(flags);
    const auto d_in = p.in(in, in_len * 32), d_out = p.out(out, out_len * 32);
    return launch_batch(Counts(ctx, flags), p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_digest(limbs(tag), d_in(d), cnt, il, d_out(d), ol, truncate, ctx->coop_max,
                                                 st));
    });
}

int p252_digest_batch(p252_ctx* ctx, const p252_fr* tag, const p252_fr* in, size_t n, size_t in_len, p252_fr* out,
                      size_t out_len, int flags) {
    return digest_impl(ctx, tag, in, n, in_len, out, out_len, flags, false);
}

int p252_hash_batch(p252_ctx* ctx, int domain, const p252_fr* in, size_t n, size_t in_len, p252_fr* out,
                    size_t out_len, int flags) {
    p252_fr tag;
    int rc = p252_hash_tag(domain, in_len, out_len, &tag);
    if (rc != P252_OK) return rc;
    return digest_impl(ctx, &tag, in, n, in_len, out, out_len, flags, false);
}

int p252_hash_batch_truncated(p252_ctx* ctx, int domain, const p252_fr* in, size_t n, size_t in_len, p252_fr* out_raw,
                              size_t out_len, int flags) {
    p252_fr tag;
    int rc = p252_hash_tag(domain, in_len, out_len, &tag);
    if (rc != P252_OK) return rc;
    return digest_impl(ctx, &tag, in, n, in_len, out_raw, out_len, flags, true);
}

static int convert_impl(p252_ctx* ctx, const void* in, size_t n, void* out, uint8_t* ok, int flags, bool from_bytes) {
    if (!ctx || !args_ok(n, flags, {in, out})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    Plan p(flags);
    const auto d_in = p.in(in, 32), d_out = p.out(out, 32);
    const bool with_ok = from_bytes && ok;
    const auto d_ok = with_ok ? p.out(ok, 1) : Buf<uint8_t>{};
    return launch_batch(Counts(ctx, flags), p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_convert(d_in(d), cnt, d_out(d), with_ok ? d_ok(d) : nullptr, from_bytes, st));
    });
}

int p252_scalars_from_bytes(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out, uint8_t* ok, int flags) {
    return convert_impl(ctx, bytes, n, out, ok, flags, true);
}

int p252_scalars_to_bytes(p252_ctx* ctx, const p252_fr* in, size_t n, uint8_t* bytes, int flags) {
    return convert_impl(ctx, in, n, bytes, nullptr, flags, false);
}

int p252_scalars_from_bytes_wide(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out, int flags) {
    if (!ctx || !args_ok(n, flags, {bytes, out})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    Plan p(flags);
    const auto d_bytes = p.in(bytes, 64);
    const auto d_out = p.out(out, 32);
    return launch_batch(Counts(ctx, flags), p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_from_bytes_wide(d_bytes(d), cnt, d_out(d), st));
    });
}

int p252_encrypt_batch(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_fr* secret_uv,
                       const p252_fr* nonce, p252_fr* cipher, int flags) {
    if (!ctx || ((!msg || !secret_uv || !nonce || !cipher) && n)) return P252_ERR_INVALID_ARGUMENT;
    p252_fr tag;
    int rc = p252_encryption_tag(L, &tag);
    if (rc != P252_OK) return rc;
    if (!args_ok(n, flags, {msg, secret_uv, nonce, cipher})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const uint32_t l32 = (uint32_t)L;
    Plan p(flags);
    const auto d_msg = p.in(msg, L * 32), d_secret = p.in(secret_uv, 64), d_nonce = p.in(nonce, 32),
               d_cipher = p.out(cipher, (L + 1) * 32);
    return launch_batch(Counts(ctx, flags), p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_encrypt(limbs(&tag), d_msg(d), cnt, l32, d_secret(d), d_nonce(d), d_cipher(d),
                                                  st));
    }, /*wipe=*/true);
}

int p252_decrypt_batch(p252_ctx* ctx, const p252_fr* cipher, size_t n, size_t L, const p252_fr* secret_uv,
                       const p252_fr* nonce, p252_fr* msg, uint8_t* ok, size_t* n_failed, int flags) {
    if (!ctx || ((!cipher || !secret_uv || !nonce || !msg || !ok) && n)) return P252_ERR_INVALID_ARGUMENT;
    p252_fr tag;
    int rc = p252_encryption_tag(L, &tag);
    if (rc != P252_OK) return rc;
    if (!args_ok(n, flags, {cipher, secret_uv, nonce, msg}, {ok})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const uint32_t l32 = (uint32_t)L;
    const Counts counts(ctx, flags, n_failed, ok, n);
    Plan p(flags);
    const auto d_cipher = p.in(cipher, (L + 1) * 32), d_secret = p.in(secret_uv, 64), d_nonce = p.in(nonce, 32),
               d_msg = p.out(msg, L * 32);
    const auto d_ok = p.out(ok, 1);
    return launch_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_decrypt(limbs(&tag), d_cipher(d), cnt, l32, d_secret(d), d_nonce(d), d_msg(d),
                                                  d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

// ---- JubJub key exchange (dhke) and the encrypt / decrypt batches that derive their shared secret with it -------------
int p252_dhke_batch(p252_ctx* ctx, const p252_jscalar* secret, size_t n_secret, const p252_fr* public_uv, size_t n_public,
                    size_t n, p252_fr* shared_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !one_or_n(n_secret, n) || !one_or_n(n_public, n) || !args_ok(n, flags, {secret, public_uv, shared_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1, pb = n_public == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    Plan p(flags);
    const auto d_secret = p.in(secret, 32, sb), d_public = p.in(public_uv, 64, pb), d_shared = p.out(shared_uv, 64);
    const auto d_ok = p.out(ok, 1);
    return launch_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_dhke(d_secret(d), sb, d_public(d), pb, cnt, d_shared(d), d_ok(d),
                                               counts.counter(0), st));
    }, /*wipe=*/true);
}

// launch_dhke into a slot arena, then the unchanged launch_encrypt / launch_decrypt on those shared secrets, then
// launch_dhke_fix.  The shared secrets live only in the slot arenas for BOTH memory spaces (DEVICE buffers are used in
// place, chunk by chunk), so the common exit join_slots(wipe) clears them on every path.  count: *n_invalid (encrypt) or
// *n_failed (decrypt: authentication failures and invalid items, each once).
static int crypt_dhke(p252_ctx* ctx, bool decrypt, const p252_fr* in, size_t n, size_t L, const p252_jscalar* secret,
                      size_t n_secret, const p252_fr* public_uv, size_t n_public, const p252_fr* nonce, p252_fr* out,
                      uint8_t* ok, size_t* count, int flags) {
    if (!ctx || !one_or_n(n_secret, n) || !one_or_n(n_public, n) ||
        !args_ok(n, flags, {in, secret, public_uv, nonce, out}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    p252_fr tag;
    int rc = p252_encryption_tag(L, &tag);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1, pb = n_public == 1;
    const uint32_t l32 = (uint32_t)L, out_row = decrypt ? l32 : l32 + 1;
    const Counts counts(ctx, flags, count, ok, n);
    if (n == 0) return P252_OK;
    Plan p(flags);
    const auto d_in = p.in(in, (decrypt ? L + 1 : L) * 32), d_secret = p.in(secret, 32, sb),
               d_public = p.in(public_uv, 64, pb), d_nonce = p.in(nonce, 32), d_out = p.out(out, (size_t)out_row * 32);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        unsigned long long* counter = counts.counter(0);
        LAUNCH(p252::launch_dhke(d_secret(d), sb, d_public(d), pb, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(decrypt ? p252::launch_decrypt(limbs(&tag), d_in(d), cnt, l32, d_shared(d), d_nonce(d), d_out(d), d_ok(d),
                                              counter, st)
                       : p252::launch_encrypt(limbs(&tag), d_in(d), cnt, l32, d_shared(d), d_nonce(d), d_out(d), st));
        return launched(ctx, p252::launch_dhke_fix(decrypt, d_valid(d), cnt, d_out(d), out_row, d_ok(d), counter, st));
    }, /*wipe=*/true);
}

int p252_encrypt_batch_dhke(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_jscalar* secret, size_t n_secret,
                            const p252_fr* public_uv, size_t n_public, const p252_fr* nonce, p252_fr* cipher, uint8_t* ok,
                            size_t* n_invalid, int flags) {
    return crypt_dhke(ctx, false, msg, n, L, secret, n_secret, public_uv, n_public, nonce, cipher, ok, n_invalid, flags);
}

int p252_decrypt_batch_dhke(p252_ctx* ctx, const p252_fr* cipher, size_t n, size_t L, const p252_jscalar* secret,
                            size_t n_secret, const p252_fr* public_uv, size_t n_public, const p252_fr* nonce, p252_fr* msg,
                            uint8_t* ok, size_t* n_failed, int flags) {
    return crypt_dhke(ctx, true, cipher, n, L, secret, n_secret, public_uv, n_public, nonce, msg, ok, n_failed, flags);
}

// ---- fixed-base JubJub scalar multiplication and the sender's encrypt batch ------------------------------------------
// The base is public and arrives as a HOST pointer for every memory space: checked here before anything runs.
static int base_check(const p252_fr* base_uv) {
    return p252::host::jubjub_on_curve(base_uv[0].l, base_uv[1].l) ? P252_OK : P252_ERR_INVALID_POINT;
}

// The device table of base_uv in the cache slot t (ctx->bt, or one of ctx->bt2): the cached one when the base is the same
// 64 bytes, otherwise built on the context stream (k_fixed_base_table) into a new stream-ordered allocation.  The replaced
// table is freed in stream order, after every kernel already enqueued that reads it (DEVICE calls run on the context
// stream, HOST and fused calls join back into it), so P252_ASYNC calls with different bases may follow each other.
static int base_table(p252_ctx* ctx, BaseTable& t, const p252_fr* base_uv, const void** table) {
    if (t.dev && memcmp(t.key, base_uv, sizeof t.key) == 0) {
        *table = t.dev;
        return P252_OK;
    }
    void* d = nullptr;
    CU(cudaMallocAsync(&d, p252::kFixedBaseTableBytes, ctx->stream));
    uint64_t b[8];
    memcpy(b, base_uv, sizeof b);
    const int rc = launched(ctx, p252::launch_fixed_base_table(b, d, ctx->stream));
    if (rc != P252_OK) {
        cudaFreeAsync(d, ctx->stream);
        return rc;
    }
    void* old = t.dev;
    t.dev = d;
    memcpy(t.key, base_uv, sizeof t.key);
    *table = d;
    if (old) CU(cudaFreeAsync(old, ctx->stream));
    return P252_OK;
}

int p252_fixed_base_batch(p252_ctx* ctx, const p252_fr* base_uv, const p252_jscalar* secret, size_t n, p252_fr* out_uv,
                          uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !args_ok(n, flags, {secret, out_uv}, {ok})) return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_secret = p.in(secret, 32), d_out = p.out(out_uv, 64);
    const auto d_ok = p.out(ok, 1);
    return launch_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_fixed_base(d_secret(d), cnt, table, d_out(d), d_ok(d), counts.counter(0),
                                                     st));
    }, /*wipe=*/true);
}

// The sender: launch_fixed_base (R), launch_dhke into a slot arena (the shared secrets), the unchanged launch_encrypt,
// then launch_dhke_fix on the cipher rows and again on the R rows, so that an item with an invalid r or public key has
// ok = 0 and both rows zeroed.  As in crypt_dhke the shared secrets live only in the slot arenas, for both memory spaces,
// and the common exit join_slots(wipe) clears them on every path.
int p252_encrypt_batch_ephemeral(p252_ctx* ctx, const p252_fr* msg, size_t n, size_t L, const p252_jscalar* r,
                                 const p252_fr* base_uv, const p252_fr* public_uv, size_t n_public, const p252_fr* nonce,
                                 p252_fr* cipher, p252_fr* R_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !one_or_n(n_public, n) || !args_ok(n, flags, {msg, r, public_uv, nonce, cipher, R_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    p252_fr tag;
    int rc = p252_encryption_tag(L, &tag);
    if (rc != P252_OK || (rc = base_check(base_uv)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const uint32_t l32 = (uint32_t)L;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_msg = p.in(msg, L * 32), d_r = p.in(r, 32), d_public = p.in(public_uv, 64, pb),
               d_nonce = p.in(nonce, 32), d_cipher = p.out(cipher, (size_t)(l32 + 1) * 32), d_R = p.out(R_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_dhke(d_r(d), false, d_public(d), pb, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_encrypt(limbs(&tag), d_msg(d), cnt, l32, d_shared(d), d_nonce(d), d_cipher(d), st));
        LAUNCH(p252::launch_dhke_fix(false, d_valid(d), cnt, d_cipher(d), l32 + 1, d_ok(d), counts.counter(0), st));
        return launched(ctx, p252::launch_dhke_fix(false, d_valid(d), cnt, d_R(d), 2, d_ok(d), nullptr, st));
    }, /*wipe=*/true);
}

// ---- stealth addresses: the sender's (R, note_pk) and the receiver's ownership scan ----------------------------------
// hash(P) = Hash::digest_truncated(Domain::Other, [P.u, P.v])[0].  Sender: R = [r] G, note_pk = [hash([r] A)] G + B;
// receiver (view key a, spend key B): owns <=> note_pk == [hash([a] R)] G + B.  Per chunk: launch_dhke into a slot arena
// (the shared points and their validity), the truncated launch_digest of them into the arena (h), then launch_stealth_*
// (the sender runs launch_fixed_base for R first).  r, view_a, the shared points and h live only in the slot arenas for
// both memory spaces, so both calls are synchronous and the common exit join_slots(wipe) clears them on every path.
static int stealth_tag(p252_fr* tag) { return p252_hash_tag(P252_DOMAIN_OTHER, 2, 1, tag); }

int p252_stealth_address_batch(p252_ctx* ctx, const p252_jscalar* r, size_t n, const p252_fr* base_uv, const p252_fr* A_uv,
                               const p252_fr* B_uv, size_t n_public, p252_fr* R_uv, p252_fr* note_pk_uv, uint8_t* ok,
                               size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !one_or_n(n_public, n) || !args_ok(n, flags, {r, A_uv, B_uv, R_uv, note_pk_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    p252_fr tag;
    if (rc != P252_OK || (rc = stealth_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_r = p.in(r, 32), d_A = p.in(A_uv, 64, pb), d_B = p.in(B_uv, 64, pb), d_R = p.out(R_uv, 64),
               d_note_pk = p.out(note_pk_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_dhke(d_r(d), false, d_A(d), pb, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_stealth_derive(d_h(d), cnt, table, d_B(d), pb, d_valid(d), d_R(d),
                                                         d_note_pk(d), d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

// The receiver's B is public and a HOST pointer, like the base: checked here, and its Niels form computed once on the host
// and passed to the kernel by value.  An item's owned flag does not tell an invalid item from a note of someone else, so
// both counts come from the device counters (0: owned, 1: invalid) for both memory spaces.
int p252_stealth_owns_batch(p252_ctx* ctx, const p252_jscalar* view_a, const p252_fr* spend_B_uv, const p252_fr* base_uv,
                            const p252_fr* R_uv, const p252_fr* note_pk_uv, size_t n, uint8_t* owned, size_t* n_owned,
                            size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !spend_B_uv || !args_ok(n, flags, {view_a, R_uv, note_pk_uv}, {owned}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(base_uv)) != P252_OK || (rc = base_check(spend_B_uv)) != P252_OK) return rc;
    p252_fr tag;
    if ((rc = stealth_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts = Counts::device(ctx, flags, n_owned, n_invalid);
    if (n == 0) return P252_OK;
    uint64_t nb[12];
    p252::host::jubjub_niels(nb, spend_B_uv[0].l, spend_B_uv[1].l);
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(view_a, 32, true), d_R = p.in(R_uv, 64), d_note_pk = p.in(note_pk_uv, 64);
    const auto d_owned = p.out(owned, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_dhke(d_a(d), true, d_R(d), false, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_stealth_owns(d_h(d), cnt, table, nb, d_note_pk(d), d_valid(d), d_owned(d),
                                                       counts.counter(0), counts.counter(1), st));
    }, /*wipe=*/true);
}

// ---- Schnorr signatures over JubJub: signing and verification ----------------------------------------------------------
// challenge(R, m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, m])[0].  Sign: R = [r] G, u = (r - c sk) mod r_J;
// verify: [u] G + [c] PK == R.  Per chunk: launch_schnorr_pack writes the rows [R.u, R.v, m] into a slot arena, the
// truncated launch_digest of them gives c into the arena, then launch_schnorr_sign / launch_schnorr_verify (the signer runs
// launch_fixed_base for R first).  Signing stages sk and r only in the slot arenas (DEVICE buffers are used in place), so
// it is synchronous and the common exit join_slots(wipe) clears them on every path; verification reads public data only.
static int schnorr_tag(p252_fr* tag) { return p252_hash_tag(P252_DOMAIN_OTHER, 3, 1, tag); }

int p252_schnorr_sign_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_jscalar* r, const p252_fr* msg,
                            size_t n, const p252_fr* base_uv, p252_jscalar* u_out, p252_fr* R_uv, uint8_t* ok, size_t* n_invalid,
                            int flags) {
    if (!ctx || !base_uv || !one_or_n(n_secret, n) || !args_ok(n, flags, {sk, r, msg, u_out, R_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    p252_fr tag;
    if (rc != P252_OK || (rc = schnorr_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_sk = p.in(sk, 32, sb), d_r = p.in(r, 32), d_msg = p.in(msg, 32), d_u = p.out(u_out, 32),
               d_R = p.out(R_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_rows = p.arena(96), d_c = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_schnorr_pack(d_R(d), d_msg(d), cnt, d_rows(d), d_ok(d), true, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 3, d_c(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_schnorr_sign(d_sk(d), sb, d_r(d), d_c(d), cnt, d_u(d), d_R(d), d_ok(d),
                                                       counts.counter(0), st));
    }, /*wipe=*/true);
}

// An item's verified flag does not tell an invalid item from a signature that does not verify, so both counts come from
// the device counters (0: verified, 1: invalid) for both memory spaces.  Nothing here is secret: no wipe.
int p252_schnorr_verify_batch(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_jscalar* u, const p252_fr* R_uv,
                              const p252_fr* msg, size_t n, const p252_fr* base_uv, uint8_t* verified, size_t* n_verified,
                              size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !one_or_n(n_public, n) || !args_ok(n, flags, {pk_uv, u, R_uv, msg}, {verified}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    p252_fr tag;
    if (rc != P252_OK || (rc = schnorr_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts = Counts::device(ctx, flags, n_verified, n_invalid);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_pk = p.in(pk_uv, 64, pb), d_u = p.in(u, 32), d_R = p.in(R_uv, 64), d_msg = p.in(msg, 32);
    const auto d_verified = p.out(verified, 1);
    const auto d_rows = p.arena(96);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_c = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_schnorr_pack(d_R(d), d_msg(d), cnt, d_rows(d), d_valid(d), false, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 3, d_c(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_schnorr_verify(d_pk(d), pb, d_u(d), d_R(d), d_c(d), d_valid(d), cnt, table,
                                                         d_verified(d), counts.counter(0), counts.counter(1), st));
    });
}

// ---- note nullifiers: Hash::digest(Domain::Other, [pk'.u, pk'.v, pos])[0], pk' = [(hash([a] R) + b) mod r_J] G' --------
// Per chunk: launch_dhke into a slot arena (the shared points and their validity), the truncated launch_digest of them
// into the arena (h, the stealth calls' hash), launch_nullifier_key (the digest rows [pk'.u, pk'.v, pos] into the arena,
// validity &= b < r_J), the full launch_digest of the rows into nullifier (the Schnorr challenge's tag: Domain::Other,
// three inputs, one output), then launch_dhke_fix (invalid rows zeroed, ok, the count).  a, b, the shared points, h,
// note_sk and pk' live only in the slot arenas for both memory spaces, so the call is synchronous and the common exit
// join_slots(wipe) clears them on every path.
int p252_nullifier_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret, const p252_fr* base_uv,
                         const p252_fr* R_uv, const uint64_t* pos, size_t n, p252_fr* nullifier, uint8_t* ok,
                         size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !one_or_n(n_secret, n) || !args_ok(n, flags, {a, b, R_uv, nullifier}, {ok}, {pos}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    p252_fr tag_h, tag_n;
    if (rc != P252_OK || (rc = stealth_tag(&tag_h)) != P252_OK || (rc = schnorr_tag(&tag_n)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(a, 32, sb), d_b = p.in(b, 32, sb), d_R = p.in(R_uv, 64);
    const auto d_pos = p.in(pos, 8);
    const auto d_nullifier = p.out(nullifier, 32);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32), d_rows = p.arena(96);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_dhke(d_a(d), sb, d_R(d), false, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag_h), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        LAUNCH(p252::launch_nullifier_key(d_h(d), d_b(d), sb, d_pos(d), cnt, table, d_rows(d), d_valid(d), st));
        LAUNCH(p252::launch_digest(limbs(&tag_n), d_rows(d), cnt, 3, d_nullifier(d), 1, false, ctx->coop_max, st));
        return launched(ctx, p252::launch_dhke_fix(false, d_valid(d), cnt, d_nullifier(d), 1, d_ok(d),
                                                   counts.counter(0), st));
    }, /*wipe=*/true);
}

// ---- double-key Schnorr signatures over G and G' (jubjub-schnorr SignatureDouble) and note signing ----------------------
// challenge2(R, R', m) = Hash::digest_truncated(Domain::Other, [R.u, R.v, R'.u, R'.v, m])[0].  Sign: R = [r] G, R' = [r] G',
// u = (r - c sk) mod r_J; verify: [u] G + [c] PK == R and [u] G' + [c] PK' == R'.  The note signer's key is
// note_sk = (hash([a] R_note) + b) mod r_J, and it also returns pk' = [note_sk] G'.  Per chunk: launch_fixed_base twice on
// the same r (R with the table of G, R' with the table of G'; both write the same ok), launch_schnorr_pack_double writes
// the rows [R.u, R.v, R'.u, R'.v, m] into a slot arena, the truncated launch_digest of them gives c into the arena, then
// launch_schnorr_sign_double / launch_note_sign_double / launch_schnorr_verify_double.  The note signer first runs
// launch_dhke and the truncated launch_digest of the shared points (h, the stealth calls' hash) into the arena, as the
// nullifier call does.  The secrets (sk, r, a, b, [a] R_note, h, note_sk) live only in the slot arenas for both memory
// spaces, so both signing calls are synchronous and the common exit join_slots(wipe) clears them on every path;
// verification reads public data only.  The tables of G and G' come from the context's two-slot cache ctx->bt2.
static int schnorr_double_tag(p252_fr* tag) { return p252_hash_tag(P252_DOMAIN_OTHER, 5, 1, tag); }

static int double_tables(p252_ctx* ctx, const p252_fr* G_uv, const p252_fr* Gp_uv, const void** table, const void** table_p) {
    const int rc = base_table(ctx, ctx->bt2[0], G_uv, table);
    return rc != P252_OK ? rc : base_table(ctx, ctx->bt2[1], Gp_uv, table_p);
}

int p252_schnorr_sign_double_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_jscalar* r,
                                   const p252_fr* msg, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, p252_jscalar* u_out,
                                   p252_fr* R_uv, p252_fr* Rp_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !one_or_n(n_secret, n) || !args_ok(n, flags, {sk, r, msg, u_out, R_uv, Rp_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag;
    if ((rc = schnorr_double_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_sk = p.in(sk, 32, sb), d_r = p.in(r, 32), d_msg = p.in(msg, 32), d_u = p.out(u_out, 32),
               d_R = p.out(R_uv, 64), d_Rp = p.out(Rp_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_rows = p.arena(160), d_c = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table_p, d_Rp(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_schnorr_pack_double(d_R(d), d_Rp(d), d_msg(d), cnt, d_rows(d), d_ok(d), true, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 5, d_c(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_schnorr_sign_double(d_sk(d), sb, d_r(d), d_c(d), cnt, d_u(d), d_R(d), d_Rp(d),
                                                              d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

// As p252_schnorr_verify_batch, both counts come from the device counters (0: verified, 1: invalid) for both memory
// spaces, and nothing here is secret: no wipe.
int p252_schnorr_verify_double_batch(p252_ctx* ctx, const p252_fr* pk_uv, const p252_fr* pkp_uv, size_t n_public,
                                     const p252_jscalar* u, const p252_fr* R_uv, const p252_fr* Rp_uv, const p252_fr* msg,
                                     size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, uint8_t* verified, size_t* n_verified,
                                     size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !one_or_n(n_public, n) ||
        !args_ok(n, flags, {pk_uv, pkp_uv, u, R_uv, Rp_uv, msg}, {verified}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag;
    if ((rc = schnorr_double_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts = Counts::device(ctx, flags, n_verified, n_invalid);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_pk = p.in(pk_uv, 64, pb), d_pkp = p.in(pkp_uv, 64, pb), d_u = p.in(u, 32), d_R = p.in(R_uv, 64),
               d_Rp = p.in(Rp_uv, 64), d_msg = p.in(msg, 32);
    const auto d_verified = p.out(verified, 1);
    const auto d_rows = p.arena(160);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_c = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_schnorr_pack_double(d_R(d), d_Rp(d), d_msg(d), cnt, d_rows(d), d_valid(d), false, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 5, d_c(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_schnorr_verify_double(d_pk(d), d_pkp(d), pb, d_u(d), d_R(d), d_Rp(d), d_c(d),
                                                                d_valid(d), cnt, table, table_p, d_verified(d),
                                                                counts.counter(0), counts.counter(1), st));
    });
}

int p252_note_sign_double_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret,
                                const p252_fr* note_R_uv, const p252_jscalar* r, const p252_fr* msg, size_t n,
                                const p252_fr* G_uv, const p252_fr* Gp_uv, p252_jscalar* u_out, p252_fr* R_uv, p252_fr* Rp_uv,
                                p252_fr* pkp_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !one_or_n(n_secret, n) ||
        !args_ok(n, flags, {a, b, note_R_uv, r, msg, u_out, R_uv, Rp_uv, pkp_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag_h, tag;
    if ((rc = stealth_tag(&tag_h)) != P252_OK || (rc = schnorr_double_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(a, 32, sb), d_b = p.in(b, 32, sb), d_note_R = p.in(note_R_uv, 64), d_r = p.in(r, 32),
               d_msg = p.in(msg, 32), d_u = p.out(u_out, 32), d_R = p.out(R_uv, 64), d_Rp = p.out(Rp_uv, 64),
               d_pkp = p.out(pkp_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32), d_rows = p.arena(160), d_c = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_dhke(d_a(d), sb, d_note_R(d), false, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag_h), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table_p, d_Rp(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_schnorr_pack_double(d_R(d), d_Rp(d), d_msg(d), cnt, d_rows(d), d_ok(d), true, st));
        LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 5, d_c(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_note_sign_double(d_b(d), sb, d_h(d), d_valid(d), d_r(d), d_c(d), cnt, table_p,
                                                           d_u(d), d_R(d), d_Rp(d), d_pkp(d), d_ok(d),
                                                           counts.counter(0), st));
    }, /*wipe=*/true);
}

// ---- note values: commitments C = [v] G + [blinder] G', creating obfuscated notes and opening them ----------------------
// commit: one launch_value_commit per chunk.  create (the sender): launch_fixed_base (R), launch_dhke (the shared point
// S = [r] A into a slot arena), the truncated launch_digest of S (h, the stealth calls' hash), launch_note_value (C, the
// message rows [Fr(v), Fr(blinder)] into the arena, validity &= blinder < r_J), launch_stealth_derive (note_pk; it zeroes R
// of an invalid item, sets ok and counts), launch_encrypt at L = 2 with S, then launch_dhke_fix on the cipher rows and again
// on the commitment rows.  Both fixes read ok as the validity, because only ok holds every check (B's is made by
// launch_stealth_derive); they count nothing.  open (the wallet): launch_dhke (S = [a] R), launch_decrypt at L = 2 into the
// arena (no count), launch_note_open_value (range checks, the commitment check, outputs, ok and the count of every item
// that did not open).  The secrets (r, v, blinder, a, S, h and the plaintext rows) live only in the slot arenas for both
// memory spaces, so all three calls are synchronous and the common exit join_slots(wipe) clears them on every path.  The
// tables of G and G' come from the context's two-slot cache ctx->bt2, shared with the double-key signature calls.
int p252_value_commit_batch(p252_ctx* ctx, const uint64_t* value, const p252_jscalar* blinder, size_t n, const p252_fr* G_uv,
                            const p252_fr* Gp_uv, p252_fr* commitment_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !args_ok(n, flags, {blinder, commitment_uv}, {ok}, {value}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_value = p.in(value, 8);
    const auto d_blinder = p.in(blinder, 32), d_C = p.out(commitment_uv, 64);
    const auto d_ok = p.out(ok, 1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_value_commit(d_value(d), d_blinder(d), cnt, table, table_p, d_C(d), d_ok(d),
                                                       counts.counter(0), st));
    }, /*wipe=*/true);
}

int p252_note_create_batch(p252_ctx* ctx, const p252_jscalar* r, const uint64_t* value, const p252_jscalar* blinder,
                           const p252_fr* nonce, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, const p252_fr* A_uv,
                           const p252_fr* B_uv, size_t n_public, p252_fr* R_uv, p252_fr* note_pk_uv, p252_fr* commitment_uv,
                           p252_fr* cipher, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !one_or_n(n_public, n) ||
        !args_ok(n, flags, {r, blinder, nonce, A_uv, B_uv, R_uv, note_pk_uv, commitment_uv, cipher}, {ok}, {value}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag_h, tag_e;
    if ((rc = stealth_tag(&tag_h)) != P252_OK || (rc = p252_encryption_tag(2, &tag_e)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_r = p.in(r, 32);
    const auto d_value = p.in(value, 8);
    const auto d_blinder = p.in(blinder, 32), d_nonce = p.in(nonce, 32), d_A = p.in(A_uv, 64, pb),
               d_B = p.in(B_uv, 64, pb), d_R = p.out(R_uv, 64), d_note_pk = p.out(note_pk_uv, 64),
               d_C = p.out(commitment_uv, 64), d_cipher = p.out(cipher, 96);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32), d_rows = p.arena(64);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_fixed_base(d_r(d), cnt, table, d_R(d), d_ok(d), nullptr, st));
        LAUNCH(p252::launch_dhke(d_r(d), false, d_A(d), pb, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag_h), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        LAUNCH(p252::launch_note_value(d_value(d), d_blinder(d), cnt, table, table_p, d_C(d), d_rows(d), d_valid(d),
                                       st));
        LAUNCH(p252::launch_stealth_derive(d_h(d), cnt, table, d_B(d), pb, d_valid(d), d_R(d), d_note_pk(d), d_ok(d),
                                           counts.counter(0), st));
        LAUNCH(p252::launch_encrypt(limbs(&tag_e), d_rows(d), cnt, 2, d_shared(d), d_nonce(d), d_cipher(d), st));
        LAUNCH(p252::launch_dhke_fix(false, d_ok(d), cnt, d_cipher(d), 3, d_ok(d), nullptr, st));
        return launched(ctx, p252::launch_dhke_fix(false, d_ok(d), cnt, d_C(d), 2, d_ok(d), nullptr, st));
    }, /*wipe=*/true);
}

int p252_note_open_batch(p252_ctx* ctx, const p252_jscalar* a, size_t n_secret, const p252_fr* R_uv, const p252_fr* nonce,
                         const p252_fr* cipher, const p252_fr* commitment_uv, size_t n, const p252_fr* G_uv,
                         const p252_fr* Gp_uv, uint64_t* value, p252_jscalar* blinder, uint8_t* ok, size_t* n_failed,
                         int flags) {
    if (!ctx || !G_uv || !Gp_uv || !one_or_n(n_secret, n) ||
        !args_ok(n, flags, {a, R_uv, nonce, cipher, commitment_uv, blinder}, {ok}, {value}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag_e;
    if ((rc = p252_encryption_tag(2, &tag_e)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_failed, ok, n);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(a, 32, sb), d_R = p.in(R_uv, 64), d_nonce = p.in(nonce, 32), d_cipher = p.in(cipher, 96),
               d_C = p.in(commitment_uv, 64);
    const auto d_value = p.out(value, 8);
    const auto d_blinder = p.out(blinder, 32);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_rows = p.arena(64);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_dhke(d_a(d), sb, d_R(d), false, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_decrypt(limbs(&tag_e), d_cipher(d), cnt, 2, d_shared(d), d_nonce(d), d_rows(d), d_ok(d),
                                    nullptr, st));
        return launched(ctx, p252::launch_note_open_value(d_rows(d), d_valid(d), d_C(d), cnt, table, table_p,
                                                          d_value(d), d_blinder(d), d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

// ---- multi-key wallet scans: owner, nullifier, checked opening and per-key totals of every note -----------------------
// Per chunk, first phase over the chunk's n k pairs (note i, key j at i k + j): launch_wallet_keys (the keys' B_j = [b_j] G
// in Niels form and their validity, from the a and b rows staged once per chunk), launch_wallet_dhke ([a_j] R_i), the
// truncated launch_digest of every pair's point (h, the stealth calls' hash), launch_wallet_match (the ownership check) and
// launch_wallet_select (owner, zeroed rows, the invalid count, the owned notes compacted into dense rows).  The host then
// reads the chunk's owned count (one synchronise per chunk, run_host_pipeline2: after the next chunk's first phase is
// enqueued, so the chunks overlap) and the second phase runs on the owned rows only, with the nullifier call's and the opening call's unchanged kernels: launch_nullifier_key, the full launch_digest (the nullifier),
// launch_decrypt at L = 2 and launch_note_open_value; launch_wallet_scatter writes the rows back in note order and adds to
// the totals.  The keys, every shared point, its hash, note_sk, pk' and the plaintexts live only in the slot arenas for
// both memory spaces (wiped by join_slots on every path).  B_j is derived per chunk, in the chunk's arena, so that it is
// never outside a wiped arena: k fixed-base walks per chunk.  The totals accumulate in the caller's buffer (DEVICE) or in
// one per-call device buffer (HOST), zeroed first, copied out once and wiped.  Counts: device counter 0 the invalid
// notes, 1 the bad keys (counted in the first chunk only).
int p252_wallet_scan_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_keys, const p252_fr* R_uv,
                           const p252_fr* note_pk_uv, const uint64_t* pos, const p252_fr* nonce, const p252_fr* cipher,
                           const p252_fr* commitment_uv, size_t n, const p252_fr* G_uv, const p252_fr* Gp_uv, int32_t* owner,
                           p252_fr* nullifier, uint64_t* value, p252_jscalar* blinder, uint8_t* opened, uint64_t* key_totals,
                           size_t* n_invalid, size_t* n_bad_keys, int flags) {
    const bool dev = (flags & P252_MEM_DEVICE) != 0;
    if (!ctx || !G_uv || !Gp_uv || n_keys == 0 || n_keys > P252_WALLET_MAX_KEYS ||
        !args_ok(n, flags, {a, b, R_uv, note_pk_uv, nonce, cipher, commitment_uv, nullifier, blinder, key_totals},
                 {owner, opened}, {pos, value}) ||
        (dev && (reinterpret_cast<uintptr_t>(owner) & 3)))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag_h, tag_n, tag_e;
    if ((rc = stealth_tag(&tag_h)) != P252_OK || (rc = schnorr_tag(&tag_n)) != P252_OK ||
        (rc = p252_encryption_tag(2, &tag_e)) != P252_OK)
        return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const uint32_t k = (uint32_t)n_keys;
    const Counts counts = Counts::device(ctx, flags, n_invalid, n_bad_keys);
    if (n == 0) return P252_OK;
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK || (rc = counts.begin()) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(a, 32 * n_keys, true), d_b = p.in(b, 32 * n_keys, true), d_R = p.in(R_uv, 64),
               d_note_pk = p.in(note_pk_uv, 64);
    const auto d_pos = p.in(pos, 8);
    const auto d_nonce = p.in(nonce, 32), d_cipher = p.in(cipher, 96), d_C = p.in(commitment_uv, 64);
    const auto d_owner = p.out(owner, 4);
    const auto d_nullifier = p.out(nullifier, 32);
    const auto d_value = p.out(value, 8);
    const auto d_blinder = p.out(blinder, 32);
    const auto d_opened = p.out(opened, 1);
    const auto d_nb = p.arena(96 * n_keys, true);
    const auto d_kvalid = p.arena<uint8_t>(n_keys, true);
    const auto d_n_own = p.arena<unsigned long long>(8, true);
    const auto d_shared = p.arena(64 * n_keys);
    const auto d_pvalid = p.arena<uint8_t>(n_keys);
    const auto d_h = p.arena(32 * n_keys);
    const auto d_matched = p.arena<uint8_t>(n_keys);
    // dn_: the dense rows of owned notes
    const auto dn_meta = p.arena(8), dn_S = p.arena(64), dn_h = p.arena(32), dn_b = p.arena(32);
    const auto dn_pos = p.arena<uint64_t>(8);
    const auto dn_nonce = p.arena(32), dn_cipher = p.arena(96), dn_C = p.arena(64);
    const auto dn_valid = p.arena<uint8_t>(1);
    const auto dn_rows = p.arena(96), dn_nullifier = p.arena(32), dn_plain = p.arena(64);
    const auto dn_ok = p.arena<uint8_t>(1);
    const auto dn_value = p.arena<uint64_t>(8);
    const auto dn_blinder = p.arena(32);
    auto scan = [&](unsigned long long* tot) -> int {
        const size_t tot_bytes = 4 * sizeof(uint64_t) * n_keys;
        CU(cudaMemsetAsync(tot, 0, tot_bytes, ctx->stream));
        bool first = true;
        int r = run_host_pipeline2(ctx, p.ios, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
            const size_t np = cnt * k;
            LAUNCH(p252::launch_wallet_keys(d_a(d), d_b(d), k, table, d_nb(d), d_kvalid(d), d_n_own(d),
                                            first ? counts.counter(1) : nullptr, st));
            first = false;
            LAUNCH(p252::launch_wallet_dhke(d_a(d), d_kvalid(d), k, d_R(d), np, d_shared(d), d_pvalid(d), st));
            LAUNCH(p252::launch_digest(limbs(&tag_h), d_shared(d), np, 2, d_h(d), 1, true, ctx->coop_max, st));
            LAUNCH(p252::launch_wallet_match(d_h(d), np, k, table, d_nb(d), d_note_pk(d), d_pvalid(d), d_matched(d),
                                             st));
            const p252::WalletRows dense{dn_meta(d),  dn_S(d),      dn_h(d), dn_b(d),    dn_pos(d),
                                         dn_nonce(d), dn_cipher(d), dn_C(d), dn_valid(d)};
            return launched(ctx, p252::launch_wallet_select(k, d_matched(d), d_shared(d), d_h(d), d_b(d), d_R(d),
                                                            d_note_pk(d), d_pos(d), d_nonce(d), d_cipher(d), d_C(d),
                                                            cnt, d_owner(d), d_nullifier(d), d_value(d), d_blinder(d),
                                                            d_opened(d), dense, d_n_own(d), counts.counter(0), st));
        }, [&](void** d, size_t, cudaStream_t st) -> int {
            unsigned long long n_own = 0;
            CU(cudaMemcpyAsync(&n_own, d_n_own(d), sizeof n_own, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            if (n_own == 0) return P252_OK;
            LAUNCH(p252::launch_nullifier_key(dn_h(d), dn_b(d), false, dn_pos(d), n_own, table_p, dn_rows(d),
                                              dn_valid(d), st));
            LAUNCH(p252::launch_digest(limbs(&tag_n), dn_rows(d), n_own, 3, dn_nullifier(d), 1, false, ctx->coop_max,
                                       st));
            LAUNCH(p252::launch_decrypt(limbs(&tag_e), dn_cipher(d), n_own, 2, dn_S(d), dn_nonce(d), dn_plain(d),
                                        dn_ok(d), nullptr, st));
            LAUNCH(p252::launch_note_open_value(dn_plain(d), dn_valid(d), dn_C(d), n_own, table, table_p, dn_value(d),
                                                dn_blinder(d), dn_ok(d), nullptr, st));
            return launched(ctx, p252::launch_wallet_scatter(dn_meta(d), dn_nullifier(d), dn_value(d), dn_blinder(d),
                                                             dn_ok(d), n_own, d_nullifier(d), d_value(d), d_blinder(d),
                                                             d_opened(d), tot, st));
        }, /*wipe=*/true);
        if (!dev) {
            if (r == P252_OK) {
                const cudaError_t ce = cudaMemcpyAsync(key_totals, tot, tot_bytes, cudaMemcpyDeviceToHost, ctx->stream);
                if (ce != cudaSuccess) r = fail_cuda(ctx, ce, "cudaMemcpyAsync");
            }
            const cudaError_t we = cudaMemsetAsync(tot, 0, tot_bytes, ctx->stream);   // the totals are the wallet's balance
            if (r == P252_OK && we != cudaSuccess) r = fail_cuda(ctx, we, "cudaMemsetAsync");
        }
        return r;
    };
    if (dev) {
        rc = scan(reinterpret_cast<unsigned long long*>(key_totals));
    } else {
        unsigned long long* tot = nullptr;
        rc = with_scratch(ctx, ctx->stream, [&](Carve& c) { tot = c.take<unsigned long long>(4 * n_keys); },
                          [&] { return scan(tot); });
    }
    return counts.end(rc);
}

// ---- JubJub ElGamal and the encrypted sender of a Phoenix note --------------------------------------------------------
// encrypt: (c1, c2) = ([r] G, M + [r] PK); decrypt: M = c2 - [sk] c1.  The sender field is two encryptions under note_pk,
// [(c1_A, c2_A), (c1_B, c2_B)], opened with note_sk = (hash([a] R) + b) mod r_J after an ownership check
// [note_sk] G == note_pk.  encrypt, sender encrypt and decrypt: one launch per chunk (launch_elgamal_encrypt,
// launch_note_sender_encrypt, launch_elgamal_decrypt).  sender decrypt: launch_dhke ([a] R and its validity into a slot
// arena), the truncated launch_digest of it (h, the stealth calls' hash) into the arena, then launch_note_sender_decrypt,
// as p252_nullifier_batch does.  r, the blinders, M, (A, B), sk, a, b, [a] R, h and note_sk live only in the slot arenas
// for both memory spaces, so all four calls are synchronous and the common exit join_slots(wipe) clears them on every
// path.  G's fixed-base table is the double-key and note calls' first cache slot (ctx->bt2[0]): after a note call with
// the same G these calls build no table, and they evict neither G' nor the single-base slot.
int p252_elgamal_encrypt_batch(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_fr* msg_uv,
                               const p252_jscalar* r, size_t n, const p252_fr* G_uv, p252_fr* c1_uv, p252_fr* c2_uv,
                               uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !one_or_n(n_public, n) || !args_ok(n, flags, {pk_uv, msg_uv, r, c1_uv, c2_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(G_uv);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt2[0], G_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_pk = p.in(pk_uv, 64, pb), d_M = p.in(msg_uv, 64), d_r = p.in(r, 32), d_c1 = p.out(c1_uv, 64),
               d_c2 = p.out(c2_uv, 64);
    const auto d_ok = p.out(ok, 1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_elgamal_encrypt(d_pk(d), pb, d_M(d), false, d_r(d), cnt, table, d_c1(d),
                                                          d_c2(d), d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

int p252_elgamal_decrypt_batch(p252_ctx* ctx, const p252_jscalar* sk, size_t n_secret, const p252_fr* c1_uv,
                               const p252_fr* c2_uv, size_t n, p252_fr* msg_uv, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !one_or_n(n_secret, n) || !args_ok(n, flags, {sk, c1_uv, c2_uv, msg_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    Plan p(flags);
    const auto d_sk = p.in(sk, 32, sb), d_c1 = p.in(c1_uv, 64), d_c2 = p.in(c2_uv, 64), d_M = p.out(msg_uv, 64);
    const auto d_ok = p.out(ok, 1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_elgamal_decrypt(d_sk(d), sb, d_c1(d), d_c2(d), cnt, d_M(d), d_ok(d),
                                                          counts.counter(0), st));
    }, /*wipe=*/true);
}

int p252_note_sender_encrypt_batch(p252_ctx* ctx, const p252_fr* note_pk_uv, const p252_fr* sender_A_uv,
                                   const p252_fr* sender_B_uv, size_t n_sender, const p252_jscalar* blinder, size_t n,
                                   const p252_fr* G_uv, p252_fr* sender_enc, uint8_t* ok, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !one_or_n(n_sender, n) ||
        !args_ok(n, flags, {note_pk_uv, sender_A_uv, sender_B_uv, blinder, sender_enc}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(G_uv);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_sender == 1;
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt2[0], G_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_note_pk = p.in(note_pk_uv, 64), d_A = p.in(sender_A_uv, 64, sb), d_B = p.in(sender_B_uv, 64, sb),
               d_blinder = p.in(blinder, 64), d_enc = p.out(sender_enc, 256);
    const auto d_ok = p.out(ok, 1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_note_sender_encrypt(d_note_pk(d), d_A(d), d_B(d), sb, d_blinder(d), cnt,
                                                              table, d_enc(d), d_ok(d), counts.counter(0), st));
    }, /*wipe=*/true);
}

int p252_note_sender_decrypt_batch(p252_ctx* ctx, const p252_jscalar* a, const p252_jscalar* b, size_t n_secret,
                                   const p252_fr* R_uv, const p252_fr* note_pk_uv, const p252_fr* sender_enc, size_t n,
                                   const p252_fr* G_uv, p252_fr* sender_A_uv, p252_fr* sender_B_uv, uint8_t* ok,
                                   size_t* n_failed, int flags) {
    if (!ctx || !G_uv || !one_or_n(n_secret, n) ||
        !args_ok(n, flags, {a, b, R_uv, note_pk_uv, sender_enc, sender_A_uv, sender_B_uv}, {ok}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(G_uv);
    p252_fr tag_h;
    if (rc != P252_OK || (rc = stealth_tag(&tag_h)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool sb = n_secret == 1;
    const Counts counts(ctx, flags, n_failed, ok, n);
    if (n == 0) return P252_OK;
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt2[0], G_uv, &table)) != P252_OK) return rc;
    Plan p(flags);
    const auto d_a = p.in(a, 32, sb), d_b = p.in(b, 32, sb), d_R = p.in(R_uv, 64), d_note_pk = p.in(note_pk_uv, 64),
               d_enc = p.in(sender_enc, 256), d_A = p.out(sender_A_uv, 64), d_B = p.out(sender_B_uv, 64);
    const auto d_ok = p.out(ok, 1);
    const auto d_shared = p.arena(64);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_h = p.arena(32);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
        LAUNCH(p252::launch_dhke(d_a(d), sb, d_R(d), false, cnt, d_shared(d), d_valid(d), nullptr, st));
        LAUNCH(p252::launch_digest(limbs(&tag_h), d_shared(d), cnt, 2, d_h(d), 1, true, ctx->coop_max, st));
        return launched(ctx, p252::launch_note_sender_decrypt(d_h(d), d_b(d), sb, d_valid(d), d_note_pk(d), d_enc(d),
                                                              cnt, table, d_A(d), d_B(d), d_ok(d), counts.counter(0),
                                                              st));
    }, /*wipe=*/true);
}

// ---- JubJub point compression: JubJubAffine::from_bytes / to_bytes -----------------------------------------------------
// One launch per chunk (launch_points_from_bytes / launch_points_to_bytes).  HOST batches stream through the slot arenas;
// DEVICE buffers are used in place.  Nothing here is secret: no wipe.  HOST calls count the invalid items from ok on the
// host, DEVICE calls on the device counter.
static int points_impl(p252_ctx* ctx, bool from_bytes, const void* in, size_t n, void* out, uint8_t* ok, size_t* n_invalid,
                       int flags) {
    if (!ctx || !args_ok(n, flags, {in, out}, {ok})) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts(ctx, flags, n_invalid, ok, n);
    if (n == 0) return P252_OK;
    Plan p(flags);
    const auto d_in = p.in(in, from_bytes ? 32 : 64), d_out = p.out(out, from_bytes ? 64 : 32);
    const auto d_ok = p.out(ok, 1);
    return staged_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        unsigned long long* counter = counts.counter(0);
        return launched(ctx, from_bytes ? p252::launch_points_from_bytes(d_in(d), cnt, d_out(d), d_ok(d), counter, st)
                                        : p252::launch_points_to_bytes(d_in(d), cnt, d_out(d), d_ok(d), counter, st));
    });
}

int p252_points_from_bytes(p252_ctx* ctx, const uint8_t* bytes, size_t n, p252_fr* out_uv, uint8_t* ok, size_t* n_invalid,
                           int flags) {
    return points_impl(ctx, true, bytes, n, out_uv, ok, n_invalid, flags);
}

int p252_points_to_bytes(p252_ctx* ctx, const p252_fr* uv, size_t n, uint8_t* bytes, uint8_t* ok, size_t* n_invalid,
                         int flags) {
    return points_impl(ctx, false, uv, n, bytes, ok, n_invalid, flags);
}

// ---- multi-scalar multiplication and all-or-nothing Schnorr verification -----------------------------------------------
// Per chunk of m rows (msm_chunk): launch_msm_prep -> CUB radix sort of the digit keys -> launch_msm_fill -> launch_msm_bucket
// until one piece is left -> launch_msm_window, whose W window sums go to the chunk's slot of a per-call array.  After the
// pipeline, launch_msm_final on the context stream adds the chunks and writes the result.  The window width c is fixed per
// call by the largest chunk (msm_bits), so every chunk's windows line up.  Chunks share nothing but the per-call arrays,
// in which each writes only its own slots.  Variable time: scalars are public.
namespace {

struct MsmScratch {
    uint4* niels;
    uint32_t *ka, *kb, *va, *vb;
    void* temp;
    size_t temp_bytes;
    uint4* buckets;
    uint32_t* ck[2];
    uint4* cp[2];
};

size_t ceil_div(size_t a, size_t b) { return (a + b - 1) / b; }

// The temporaries of one chunk of at most M rows
MsmScratch msm_layout(Carve& cv, size_t M, int c) {
    const size_t W = (size_t)p252::msm_windows(c), N = M * W, nb = W << (c - 1);
    const size_t n1 = 2 * ceil_div(N, p252::kMsmPiece), n2 = 2 * ceil_div(n1, p252::kMsmPiece);
    MsmScratch s{};
    s.niels = cv.take<uint4>(M * 6);
    s.ka = cv.take<uint32_t>(N);
    s.kb = cv.take<uint32_t>(N);
    s.va = cv.take<uint32_t>(N);
    s.vb = cv.take<uint32_t>(N);
    cub::DeviceRadixSort::SortPairs(nullptr, s.temp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)N, 0, 32);
    s.temp = cv.take<uint8_t>(s.temp_bytes);
    s.buckets = cv.take<uint4>(nb * 8);
    s.ck[0] = cv.take<uint32_t>(n1);
    s.cp[0] = cv.take<uint4>(n1 * 8);
    s.ck[1] = cv.take<uint32_t>(n2);
    s.cp[1] = cv.take<uint4>(n2 * 8);
    return s;
}

size_t msm_scratch_bytes(size_t M, int c) {
    Carve cv;
    msm_layout(cv, M, c);
    return cv.used;
}

// One chunk: m rows (scalars sc, points pt; device) into the W window sums at wsum, with the temporaries in `scratch`
// (msm_scratch_bytes(M, c), m <= M): a region of the arena of the chunk's slot, so that a chunk reuses the region of that
// slot's previous chunk in stream order.  The arenas persist with the context, so the temporaries cost no allocation per
// call; they grow each arena to about 100-145 MiB (DESIGN.md section 4).
int msm_chunk(p252_ctx* ctx, const void* sc, const void* pt, size_t m, int c, void* scratch, size_t M, uint4* wsum,
              unsigned long long* n_invalid, cudaStream_t st) {
    Carve cv{static_cast<uint8_t*>(scratch)};
    MsmScratch s = msm_layout(cv, M, c);
    const uint32_t W = (uint32_t)p252::msm_windows(c), nb = W << (c - 1), N = (uint32_t)(m * W);
    int end_bit = 0;
    while ((1u << end_bit) <= nb) ++end_bit;         // keys <= nb (the sentinel)
    LAUNCH(p252::launch_msm_prep(sc, pt, (uint32_t)m, c, s.niels, s.ka, s.va, n_invalid, st));
    CU(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.ka, s.kb, s.va, s.vb, (int)N, 0, end_bit, st));
    LAUNCH(p252::launch_msm_fill(s.buckets, nb, st));
    size_t pieces = ceil_div(N, p252::kMsmPiece);
    LAUNCH(p252::launch_msm_bucket(true, s.kb, s.vb, s.niels, N, nb, s.buckets, pieces > 1 ? s.ck[0] : nullptr, s.cp[0],
                                   st));
    for (int src = 0; pieces > 1; src ^= 1) {
        const uint32_t len = (uint32_t)(2 * pieces);
        pieces = ceil_div(len, p252::kMsmPiece);
        LAUNCH(p252::launch_msm_bucket(false, s.ck[src], nullptr, s.cp[src], len, nb, s.buckets,
                                       pieces > 1 ? s.ck[src ^ 1] : nullptr, s.cp[src ^ 1], st));
    }
    return launched(ctx, p252::launch_msm_window(s.buckets, c, wsum, st));
}

}  // namespace

int p252_jubjub_msm(p252_ctx* ctx, const p252_jscalar* scalars, const p252_fr* points_uv, size_t n, p252_fr* out_uv,
                    size_t* n_invalid, int flags) {
    if (!ctx || !out_uv || !args_ok(n, flags, {scalars, points_uv, out_uv})) return P252_ERR_INVALID_ARGUMENT;
    const bool dev = (flags & P252_MEM_DEVICE) != 0;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts = Counts::device(ctx, flags, n_invalid);
    Plan p(flags);
    // d_scratch: the chunk's MSM temporaries (one region per slot arena), sized below
    const auto d_sc = p.in(scalars, 32), d_pt = p.in(points_uv, 64), d_scratch = p.arena(0, true);
    const size_t chunk = n ? pipeline_chunk(p.ios, n) : 0;
    const int c = p252::msm_bits(std::max<size_t>(chunk, 1));
    const size_t W = (size_t)p252::msm_windows(c), max_chunks = n ? ceil_div(n, chunk) + 3 : 0;
    p[d_scratch].item_bytes = msm_scratch_bytes(chunk, c);
    int rc = counts.begin();
    if (rc != P252_OK) return rc;
    uint4* wsum = nullptr;
    uint8_t* dout = nullptr;
    rc = with_scratch(ctx, ctx->stream, [&](Carve& cv) {
        wsum = cv.take<uint4>(max_chunks * W * 8);
        dout = cv.take<uint8_t>(64);
    }, [&]() -> int {
        uint32_t k = 0;
        const int r = run_host_pipeline(ctx, p.ios, n, [&](void** d, size_t cnt, cudaStream_t st) {
            return msm_chunk(ctx, d_sc(d), d_pt(d), cnt, c, d_scratch(d), chunk, wsum + (size_t)(k++) * W * 8,
                             counts.counter(0), st);
        });
        if (r != P252_OK) return r;
        void* out = dev ? static_cast<void*>(out_uv) : dout;
        LAUNCH(p252::launch_msm_final(wsum, k, c, out, nullptr, 0, nullptr, nullptr, nullptr, nullptr, ctx->stream));
        if (!dev) CU(cudaMemcpyAsync(out_uv, dout, 64, cudaMemcpyDeviceToHost, ctx->stream));
        return P252_OK;
    });
    return counts.end(rc);   // HOST calls return with the sum and the count published
}

// challenge(R, m) as in p252_schnorr_verify_batch.  Per chunk: launch_schnorr_pack and the truncated launch_digest (c), then
// launch_msmv_prep writes the chunk's MSM rows and its sums of z u (and z c) into the arena, and msm_chunk runs on those
// rows.  launch_msm_final adds [sum z u] G from the fixed-base table (and, for one public key, [sum z c] PK), multiplies by
// the cofactor and writes the answer into device counter 1; counter 0 counts the invalid items.
int p252_schnorr_verify_all(p252_ctx* ctx, const p252_fr* pk_uv, size_t n_public, const p252_jscalar* u, const p252_fr* R_uv,
                            const p252_fr* msg, const p252_jscalar* weight, size_t n, const p252_fr* base_uv,
                            uint8_t* all_verified, size_t* n_invalid, int flags) {
    if (!ctx || !base_uv || !all_verified || !one_or_n(n_public, n) || !args_ok(n, flags, {pk_uv, u, R_uv, msg, weight}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc = base_check(base_uv);
    p252_fr tag;
    if (rc != P252_OK || (rc = schnorr_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts = Counts::device(ctx, flags, n_invalid, nullptr, all_verified);
    if (n == 0) {
        *all_verified = 1;
        return P252_OK;
    }
    const void* table = nullptr;
    if ((rc = base_table(ctx, ctx->bt, base_uv, &table)) != P252_OK) return rc;
    const size_t per = pb ? 1 : 2;   // MSM rows per item
    Plan p(flags);
    const auto d_pk = p.in(pk_uv, 64, pb), d_u = p.in(u, 32), d_R = p.in(R_uv, 64), d_msg = p.in(msg, 32),
               d_weight = p.in(weight, 32), d_rows = p.arena(96);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_c = p.arena(32), d_sc = p.arena(32 * per), d_pt = p.arena(64 * per), d_scratch = p.arena(0, true);
    const size_t chunk = pipeline_chunk(p.ios, n), M = chunk * per;
    const int c = p252::msm_bits(M);
    const size_t W = (size_t)p252::msm_windows(c), max_chunks = ceil_div(n, chunk) + 3;
    const size_t nsum = ceil_div(n, p252::kMsmItemsPerSum);
    p[d_scratch].item_bytes = msm_scratch_bytes(M, c);   // the chunk's MSM temporaries (one region per slot arena)
    if ((rc = counts.begin()) != P252_OK) return rc;
    uint4* wsum = nullptr;
    uint8_t *zsum = nullptr, *pkc = nullptr;
    uint32_t* bad = nullptr;
    rc = with_scratch(ctx, ctx->stream, [&](Carve& cv) {
        wsum = cv.take<uint4>(max_chunks * W * 8);
        zsum = cv.take<uint8_t>(nsum * 64);
        bad = cv.take<uint32_t>(1);
        pkc = cv.take<uint8_t>(64);
    }, [&]() -> int {
        CU(cudaMemsetAsync(bad, 0, sizeof(uint32_t), ctx->stream));
        if (pb) CU(cudaMemcpyAsync(pkc, pk_uv, 64, cudaMemcpyDefault, ctx->stream));
        uint32_t k = 0;
        size_t off = 0;
        const int r = run_host_pipeline(ctx, p.ios, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
            const uint32_t sum0 = (uint32_t)(off / p252::kMsmItemsPerSum);
            off += cnt;
            LAUNCH(p252::launch_schnorr_pack(d_R(d), d_msg(d), cnt, d_rows(d), d_valid(d), false, st));
            LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 3, d_c(d), 1, true, ctx->coop_max, st));
            LAUNCH(p252::launch_msmv_prep(d_pk(d), pb, d_u(d), d_R(d), d_c(d), d_weight(d), d_valid(d), (uint32_t)cnt,
                                          d_sc(d), d_pt(d), zsum, sum0, bad, counts.counter(0), st));
            return msm_chunk(ctx, d_sc(d), d_pt(d), cnt * per, c, d_scratch(d), M, wsum + (size_t)(k++) * W * 8, nullptr,
                             st);
        });
        if (r != P252_OK) return r;
        return launched(ctx, p252::launch_msm_final(wsum, k, c, nullptr, zsum, (uint32_t)nsum, table, pb ? pkc : nullptr, bad,
                                                    counts.counter(1), ctx->stream));
    });
    return counts.end(rc);   // HOST calls return with the answer and the count published
}

// challenge2(R, R', m) as in p252_schnorr_verify_double_batch.  Per chunk: launch_schnorr_pack_double and the truncated
// launch_digest (c), then launch_msmv_prep_double writes the chunk's MSM rows (4 per item, 2 for one key pair) and its
// sums of z u, z' u (and z c, z' c) into the arena, and msm_chunk runs on those rows.  launch_msmv_final_double adds
// [sum z u] G and [sum z' u] G' from the tables of the double-key slots (and, for one key pair, [sum z c] PK and
// [sum z' c] PK'), multiplies by the cofactor and writes the answer into device counter 1; counter 0 counts the invalid
// items.
int p252_schnorr_verify_double_all(p252_ctx* ctx, const p252_fr* pk_uv, const p252_fr* pkp_uv, size_t n_public,
                                   const p252_jscalar* u, const p252_fr* R_uv, const p252_fr* Rp_uv, const p252_fr* msg,
                                   const p252_jscalar* weight, const p252_jscalar* weight_p, size_t n, const p252_fr* G_uv,
                                   const p252_fr* Gp_uv, uint8_t* all_verified, size_t* n_invalid, int flags) {
    if (!ctx || !G_uv || !Gp_uv || !all_verified || !one_or_n(n_public, n) ||
        !args_ok(n, flags, {pk_uv, pkp_uv, u, R_uv, Rp_uv, msg, weight, weight_p}))
        return P252_ERR_INVALID_ARGUMENT;
    int rc;
    if ((rc = base_check(G_uv)) != P252_OK || (rc = base_check(Gp_uv)) != P252_OK) return rc;
    p252_fr tag;
    if ((rc = schnorr_double_tag(&tag)) != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const bool pb = n_public == 1;
    const Counts counts = Counts::device(ctx, flags, n_invalid, nullptr, all_verified);
    if (n == 0) {
        *all_verified = 1;
        return P252_OK;
    }
    const void *table = nullptr, *table_p = nullptr;
    if ((rc = double_tables(ctx, G_uv, Gp_uv, &table, &table_p)) != P252_OK) return rc;
    const size_t per = pb ? 2 : 4;   // MSM rows per item
    Plan p(flags);
    const auto d_pk = p.in(pk_uv, 64, pb), d_pkp = p.in(pkp_uv, 64, pb), d_u = p.in(u, 32), d_R = p.in(R_uv, 64),
               d_Rp = p.in(Rp_uv, 64), d_msg = p.in(msg, 32), d_weight = p.in(weight, 32),
               d_weight_p = p.in(weight_p, 32), d_rows = p.arena(160);
    const auto d_valid = p.arena<uint8_t>(1);
    const auto d_c = p.arena(32), d_sc = p.arena(32 * per), d_pt = p.arena(64 * per), d_scratch = p.arena(0, true);
    const size_t chunk = pipeline_chunk(p.ios, n), M = chunk * per;
    const int c = p252::msm_bits(M);
    const size_t W = (size_t)p252::msm_windows(c), max_chunks = ceil_div(n, chunk) + 3;
    const size_t nsum = ceil_div(n, p252::kMsmItemsPerSum);
    p[d_scratch].item_bytes = msm_scratch_bytes(M, c);   // the chunk's MSM temporaries (one region per slot arena)
    if ((rc = counts.begin()) != P252_OK) return rc;
    uint4* wsum = nullptr;
    uint8_t *zsum = nullptr, *pkc = nullptr;
    uint32_t* bad = nullptr;
    rc = with_scratch(ctx, ctx->stream, [&](Carve& cv) {
        wsum = cv.take<uint4>(max_chunks * W * 8);
        zsum = cv.take<uint8_t>(nsum * 128);
        bad = cv.take<uint32_t>(1);
        pkc = cv.take<uint8_t>(128);
    }, [&]() -> int {
        CU(cudaMemsetAsync(bad, 0, sizeof(uint32_t), ctx->stream));
        if (pb) {
            CU(cudaMemcpyAsync(pkc, pk_uv, 64, cudaMemcpyDefault, ctx->stream));
            CU(cudaMemcpyAsync(pkc + 64, pkp_uv, 64, cudaMemcpyDefault, ctx->stream));
        }
        uint32_t k = 0;
        size_t off = 0;
        const int r = run_host_pipeline(ctx, p.ios, n, [&](void** d, size_t cnt, cudaStream_t st) -> int {
            const uint32_t sum0 = (uint32_t)(off / p252::kMsmItemsPerSum);
            off += cnt;
            LAUNCH(p252::launch_schnorr_pack_double(d_R(d), d_Rp(d), d_msg(d), cnt, d_rows(d), d_valid(d), false, st));
            LAUNCH(p252::launch_digest(limbs(&tag), d_rows(d), cnt, 5, d_c(d), 1, true, ctx->coop_max, st));
            LAUNCH(p252::launch_msmv_prep_double(d_pk(d), d_pkp(d), pb, d_u(d), d_R(d), d_Rp(d), d_c(d), d_weight(d),
                                                 d_weight_p(d), d_valid(d), (uint32_t)cnt, d_sc(d), d_pt(d), zsum, sum0,
                                                 bad, counts.counter(0), st));
            return msm_chunk(ctx, d_sc(d), d_pt(d), cnt * per, c, d_scratch(d), M, wsum + (size_t)(k++) * W * 8, nullptr,
                             st);
        });
        if (r != P252_OK) return r;
        return launched(ctx, p252::launch_msmv_final_double(wsum, k, c, zsum, (uint32_t)nsum, table, table_p,
                                                            pb ? pkc : nullptr, bad, counts.counter(1), ctx->stream));
    });
    return counts.end(rc);   // HOST calls return with the answer and the count published
}

// ---- arity-4 Merkle tree ------------------------------------------------------------------------------
int p252_merkle4_level(p252_ctx* ctx, const p252_fr* children, size_t n_parents, p252_fr* parents, int flags) {
    return p252_hash_batch(ctx, P252_DOMAIN_MERKLE4, children, n_parents, 4, parents, 1, flags);
}

static int merkle_domain(int arity) {
    return arity == 4 ? P252_DOMAIN_MERKLE4 : (arity == 2 ? P252_DOMAIN_MERKLE2 : -1);
}

int p252_merkle_tree_nodes(int arity, size_t n_leaves, size_t* n_internal, int* n_levels) {
    if (merkle_domain(arity) < 0) return P252_ERR_INVALID_ARGUMENT;
    const size_t A = (size_t)arity;
    size_t m = n_leaves, total = 0;
    int lv = 0;
    if (m == 0) return P252_ERR_INVALID_ARGUMENT;
    while (m > 1) {
        if (m % A) return P252_ERR_IO_PATTERN_VIOLATION;   // a level that is not a multiple of the arity
        m /= A;
        total += m;
        ++lv;
    }
    if (lv == 0) return P252_ERR_INVALID_ARGUMENT;
    if (n_internal) *n_internal = total;                 // (n_leaves - 1) / (arity - 1)
    if (n_levels) *n_levels = lv;
    return P252_OK;
}

int p252_merkle4_tree_nodes(size_t n_leaves, size_t* n_internal, int* n_levels) {
    return p252_merkle_tree_nodes(4, n_leaves, n_internal, n_levels);
}

static int merkle_build_device(p252_ctx* ctx, int arity, const p252_fr* leaves, size_t n_leaves, p252_fr* nodes) {
    p252_fr tag;
    int rc = p252_hash_tag(merkle_domain(arity), (size_t)arity, 1, &tag);
    if (rc != P252_OK) return rc;
    const p252_fr* src = leaves;
    p252_fr* dst = nodes;
    for (size_t m = n_leaves / arity; m >= 1; m /= arity) {
        rc = launched(ctx, p252::launch_digest(limbs(&tag), src, m, (uint32_t)arity, dst, 1, false, ctx->coop_max, ctx->stream));
        if (rc != P252_OK) return rc;
        src = dst;
        dst += m;
        if (m == 1) break;
    }
    return P252_OK;
}

int p252_merkle_build(p252_ctx* ctx, int arity, const p252_fr* leaves, size_t n_leaves, p252_fr* nodes_out, int flags) {
    if (!ctx || !leaves || !nodes_out) return P252_ERR_INVALID_ARGUMENT;
    size_t n_internal;
    int rc = p252_merkle_tree_nodes(arity, n_leaves, &n_internal, nullptr);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(leaves) || !aligned16(nodes_out)) return P252_ERR_INVALID_ARGUMENT;
        return device_done(ctx, merkle_build_device(ctx, arity, leaves, n_leaves, nodes_out), flags);
    }
    // HOST: the first (largest) level streams through the chunked pipeline straight from the host
    // leaves; the remaining levels run on the device-resident level.
    const size_t first = n_leaves / arity;
    p252_fr* d_nodes = nullptr;
    CU(cudaMalloc(reinterpret_cast<void**>(&d_nodes), n_internal * sizeof(p252_fr)));
    p252_fr tag;
    p252_hash_tag(merkle_domain(arity), (size_t)arity, 1, &tag);
    {
        Plan p(flags);
        const auto d_leaves = p.in(leaves, (size_t)arity * 32), d_parents = p.out(nodes_out, 32);
        size_t done = 0;   // the pipeline hands chunks in order; mirror each chunk into d_nodes as well
        rc = run_host_pipeline(ctx, p.ios, first, [&](void** d, size_t cnt, cudaStream_t st) -> int {
            LAUNCH(p252::launch_digest(limbs(&tag), d_leaves(d), cnt, (uint32_t)arity, d_parents(d), 1, false,
                                       ctx->coop_max, st));
            CU(cudaMemcpyAsync(d_nodes + done, d_parents(d), cnt * sizeof(p252_fr), cudaMemcpyDeviceToDevice, st));
            done += cnt;
            return P252_OK;
        });
    }
    if (rc == P252_OK && first > 1) {
        rc = merkle_build_device(ctx, arity, d_nodes, first, d_nodes + first);
        if (rc == P252_OK) {
            cudaError_t e = cudaMemcpyAsync(nodes_out + first, d_nodes + first, (n_internal - first) * sizeof(p252_fr),
                                            cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            if (e != cudaSuccess) rc = fail_cuda(ctx, e, "merkle D2H");
        }
    }
    cudaFree(d_nodes);
    return rc;
}

int p252_merkle4_build(p252_ctx* ctx, const p252_fr* leaves, size_t n_leaves, p252_fr* nodes_out, int flags) {
    return p252_merkle_build(ctx, 4, leaves, n_leaves, nodes_out, flags);
}

// ---- Merkle openings ----------------------------------------------------------------------------------------
static int tree_depth(int arity, size_t n_leaves, int* depth) {
    int lv = 0;
    int rc = p252_merkle_tree_nodes(arity, n_leaves, nullptr, &lv);
    if (rc != P252_OK) return rc;
    *depth = lv;
    return P252_OK;
}

int p252_merkle_open_batch(p252_ctx* ctx, int arity, const p252_fr* leaves, size_t n_leaves, const p252_fr* nodes,
                           const uint64_t* leaf_idx, size_t n, p252_fr* paths_out, int flags) {
    if (!ctx || !leaves || !nodes || ((!leaf_idx || !paths_out) && n)) return P252_ERR_INVALID_ARGUMENT;
    int depth = 0;
    int rc = tree_depth(arity, n_leaves, &depth);
    if (rc != P252_OK) return rc;
    p252::OpenLevels lv{};                              // the dense layout: full levels, packed bottom-up
    lv.m[0] = n_leaves;
    for (int l = 1; l < depth; ++l) {
        lv.m[l] = lv.m[l - 1] / (uint64_t)arity;
        lv.off[l] = (l == 1) ? 0 : lv.off[l - 1] + lv.m[l - 1];
    }
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(leaves) || !aligned16(nodes) || !aligned16(paths_out) || (reinterpret_cast<uintptr_t>(leaf_idx) & 7))
            return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        return device_done(ctx, launched(ctx, p252::launch_merkle_open(leaves, nodes, leaf_idx, n, arity, (uint32_t)depth, lv,
                                                                       paths_out, ctx->stream)), flags);
    }
    // HOST tree: an opening is a pure gather of 32-byte items the caller already holds in host memory -- shipping
    // the whole tree to the GPU to copy depth*arity scalars back would only add PCIe traffic.  No hashing happens here.
    for (size_t i = 0; i < n; ++i)
        if (leaf_idx[i] >= n_leaves) return P252_ERR_INVALID_ARGUMENT;
    open_host(leaves, nodes, leaf_idx, n, arity, depth, lv, paths_out);
    return P252_OK;
}

int p252_merkle_verify_batch(p252_ctx* ctx, int arity, int depth, const p252_fr* leaf_items, const uint64_t* leaf_idx,
                             const p252_fr* paths, const p252_fr* root, size_t n, uint8_t* ok, size_t* n_failed,
                             int flags) {
    if (!ctx || !root || !args_ok(n, flags, {leaf_items, paths}, {ok}, {leaf_idx})) return P252_ERR_INVALID_ARGUMENT;
    if (merkle_domain(arity) < 0 || depth < 1 || depth > 64) return P252_ERR_INVALID_ARGUMENT;
    p252_fr tag;
    int rc = p252_hash_tag(merkle_domain(arity), (size_t)arity, 1, &tag);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const Counts counts(ctx, flags, n_failed, ok, n);
    const size_t path_bytes = (size_t)depth * (size_t)arity * 32;
    Plan p(flags);
    const auto d_leaf = p.in(leaf_items, 32);
    const auto d_idx = p.in(leaf_idx, 8);
    const auto d_paths = p.in(paths, path_bytes);
    const auto d_ok = p.out(ok, 1);
    return launch_batch(counts, p, n, [&](void** d, size_t cnt, cudaStream_t st) {
        return launched(ctx, p252::launch_merkle_verify(limbs(&tag), limbs(root), d_leaf(d), d_idx(d), d_paths(d), cnt,
                                                        arity, (uint32_t)depth, d_ok(d), counts.counter(0), st));
    });
}

}  // extern "C"

// ---- fixed-height trees (p252_mtree) ----------------------------------------------------------------------------
namespace {

struct MLayout {
    uint64_t slots[p252::kMaxDepth + 1];   // slots of level l (0 = leaves)
    uint64_t off[p252::kMaxDepth + 1];     // first slot of level l >= 1 inside nodes; off[0] = 0
    uint64_t node_slots;
};

int mtree_layout(int arity, int height, uint64_t capacity, MLayout* L) {
    if (merkle_domain(arity) < 0 || height < 1 || height > p252::kMaxDepth || capacity == 0) return P252_ERR_INVALID_ARGUMENT;
    if (capacity > (1ull << 58)) return P252_ERR_INVALID_ARGUMENT;   // the leaf buffer's byte size must fit 64 bits
    const uint64_t A = (uint64_t)arity;
    uint64_t c = capacity, acc = 0;                                   // c = ceil(capacity / A^l)
    for (int l = 0; l < height; ++l) {
        L->slots[l] = (c + A - 1) / A * A;                             // whole groups only
        L->off[l] = l ? acc : 0;
        if (l) acc += L->slots[l];
        c = (c + A - 1) / A;
    }
    if (c != 1) return P252_ERR_INVALID_ARGUMENT;                     // capacity > A^height
    L->slots[height] = 1;
    L->off[height] = acc;
    L->node_slots = acc + 1;
    return P252_OK;
}

// occupied nodes per level: m[l] = ceil(n / A^l)
void mtree_prefix(int arity, int height, uint64_t n, uint64_t* m) {
    m[0] = n;
    for (int l = 1; l <= height; ++l) m[l] = (m[l - 1] + (uint64_t)arity - 1) / (uint64_t)arity;
}

int mtree_check(const p252_mtree* t, int flags, MLayout* L) {
    if (!t || t->struct_size < sizeof(p252_mtree) || !t->leaves || !t->nodes) return P252_ERR_INVALID_ARGUMENT;
    int rc = mtree_layout(t->arity, t->height, t->capacity, L);
    if (rc != P252_OK) return rc;
    if (t->n_leaves > t->capacity) return P252_ERR_INVALID_ARGUMENT;
    if ((flags & P252_MEM_DEVICE) && (!aligned16(t->leaves) || !aligned16(t->nodes))) return P252_ERR_INVALID_ARGUMENT;
    return P252_OK;
}

// Every level is one launch_digest over its occupied groups (the zero padding of partial groups is already in memory);
// the slots beyond each prefix are zeroed.
int mtree_build_device(p252_ctx* ctx, const MLayout& L, int arity, int height, uint64_t n, p252_fr* leaves, p252_fr* nodes) {
    p252_fr tag;
    p252_hash_tag(merkle_domain(arity), (size_t)arity, 1, &tag);
    CU(cudaMemsetAsync(leaves + n, 0, (L.slots[0] - n) * sizeof(p252_fr), ctx->stream));
    uint64_t m[p252::kMaxDepth + 1];
    mtree_prefix(arity, height, n, m);
    const p252_fr* below = leaves;
    for (int l = 1; l <= height; ++l) {
        p252_fr* level = nodes + L.off[l];
        int rc;
        if (m[l] && (rc = launched(ctx, p252::launch_digest(limbs(&tag), below, m[l], (uint32_t)arity, level, 1, false,
                                                             ctx->coop_max, ctx->stream))) != P252_OK)
            return rc;
        CU(cudaMemsetAsync(level + m[l], 0, (L.slots[l] - m[l]) * sizeof(p252_fr), ctx->stream));
        below = level;
    }
    return P252_OK;
}

// The climb of every fixed-height tree (DEVICE pointers): level l's dirty set D_l = DeviceSelect::Flagged over the
// candidates (parent, flag) of the level below -- bound[l-1] of them, count cnt[l] on the device -- then the digest of
// exactly those groups, then the candidates of the next level.  present (p252_smtree, null for p252_mtree): presence bytes
// laid out like the scalars (leaves, then nodes), kept by the presence-aware digest.
int tree_climb(p252_ctx* ctx, int A, int H, const MLayout& L, const p252_fr* leaves, p252_fr* nodes, uint8_t* present,
               uint8_t* flag, uint64_t* parent, uint64_t* d, int* cnt, const uint64_t* bound, void* cub_tmp, size_t cub_bytes) {
    p252_fr tag;
    p252_hash_tag(merkle_domain(A), (size_t)A, 1, &tag);
    const p252_fr* below = leaves;
    const uint8_t* below_p = present;
    for (int l = 1; l <= H; ++l) {
        size_t b = cub_bytes;
        CU(cub::DeviceSelect::Flagged(cub_tmp, b, parent, flag, d, cnt + l, (int)bound[l - 1], ctx->stream));
        p252_fr* level = nodes + L.off[l];
        uint8_t* level_p = present ? present + L.slots[0] + L.off[l] : nullptr;
        int rc = launched(ctx, p252::launch_mtree_digest(limbs(&tag), below, A, level, d, cnt + l, bound[l], ctx->coop_max,
                                                         ctx->stream, below_p, level_p));
        if (rc == P252_OK && l < H)
            rc = launched(ctx, p252::launch_mtree_parents(d, cnt + l, (uint32_t)bound[l], A, flag, parent, ctx->stream));
        if (rc != P252_OK) return rc;
        below = level;
        below_p = level_p;
    }
    return P252_OK;
}

// DEVICE update of a fixed-height tree: keys_launch(keys, bpos, rejected) writes each item's key (its position, or a
// sentinel below 2^end_bit that sorts last) -> stable radix sort of (key, batch position) -> write_launch(skeys, sbpos,
// flag, parent) applies the last item per position and emits the level-1 candidates -> climb, bound[l] >= |D_l|.
// Temporaries are one stream-ordered allocation; the dirty-set counts stay on the device.
template <typename Keys, typename Write>
int tree_update_device(p252_ctx* ctx, int A, int H, const MLayout& L, const p252_fr* leaves, p252_fr* nodes, uint8_t* present,
                       uint32_t n, int end_bit, const uint64_t* bound, size_t* n_rejected, Keys keys_launch, Write write_launch) {
    size_t sort_bytes = 0, select_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                       (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, end_bit, ctx->stream));
    CU(cub::DeviceSelect::Flagged(nullptr, select_bytes, (const uint64_t*)nullptr, (const uint8_t*)nullptr, (uint64_t*)nullptr,
                                  (int*)nullptr, (int)n, ctx->stream));
    const size_t cub_bytes = std::max(sort_bytes, select_bytes);
    uint64_t *keys = nullptr, *skeys = nullptr, *parent = nullptr;
    uint32_t *bpos = nullptr, *sbpos = nullptr;
    uint8_t* flag = nullptr;
    int* cnt = nullptr;
    void* cub_tmp = nullptr;
    auto layout = [&](Carve& c) {
        keys = c.take<uint64_t>(n);                        // unsorted keys, then the dirty set D_l
        skeys = c.take<uint64_t>(n);
        parent = c.take<uint64_t>(n);
        bpos = c.take<uint32_t>(n);
        sbpos = c.take<uint32_t>(n);
        flag = c.take<uint8_t>(n);
        cnt = c.take<int>(H + 1);
        cub_tmp = c.take<uint8_t>(cub_bytes);
    };
    return with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        int rc;
        if (n_rejected && (rc = counter_begin(ctx)) != P252_OK) return rc;
        if ((rc = launched(ctx, keys_launch(keys, bpos, n_rejected ? ctx->d_counter : nullptr))) != P252_OK) return rc;
        size_t b = cub_bytes;
        CU(cub::DeviceRadixSort::SortPairs(cub_tmp, b, keys, skeys, bpos, sbpos, (int)n, 0, end_bit, ctx->stream));
        if ((rc = launched(ctx, write_launch(skeys, sbpos, flag, parent))) != P252_OK) return rc;
        rc = tree_climb(ctx, A, H, L, leaves, nodes, present, flag, parent, keys, cnt, bound, cub_tmp, cub_bytes);
        return rc != P252_OK ? rc : counter_end(ctx, n_rejected);
    });
}

// smallest end_bit with key >> end_bit == 0 (at least 1): the radix sort's bit range for keys <= key
int sort_bits(uint64_t key) {
    int end_bit = 1;
    while (end_bit < 64 && (key >> end_bit)) ++end_bit;
    return end_bit;
}

// HOST updates: the batch positions of the last item per distinct index, in ascending index order (a later item on the
// same index wins) ...
std::vector<uint32_t> last_per_index(const uint64_t* idx, size_t n) {
    std::vector<uint32_t> ord(n);
    for (size_t i = 0; i < n; ++i) ord[i] = (uint32_t)i;
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return idx[a] < idx[b]; });
    size_t k = 0;
    for (size_t i = 0; i < n; ++i)
        if (i + 1 == n || idx[ord[i + 1]] != idx[ord[i]]) ord[k++] = ord[i];
    ord.resize(k);
    return ord;
}

// ... and one level up: the sorted dirty set d becomes its distinct parents d / A
void parents_host(std::vector<uint64_t>& d, uint64_t A) {
    size_t k = 0;
    for (size_t i = 0; i < d.size(); ++i)
        if (k == 0 || d[k - 1] != d[i] / A) d[k++] = d[i] / A;
    d.resize(k);
}

// HOST update: sort and dedupe here, then per level gather the dirty groups into staging, hash them through the
// staged pipeline (p252_hash_batch) and scatter the parents back.
int mtree_update_host(p252_ctx* ctx, p252_mtree* t, const MLayout& L, const uint64_t* idx, const p252_fr* values,
                      size_t n_upd, const p252_fr* append, size_t n_append) {
    const uint64_t A = (uint64_t)t->arity, n_old = t->n_leaves;
    std::vector<uint64_t> d;
    d.reserve(n_upd + n_append);
    for (uint32_t i : last_per_index(idx, n_upd)) {
        t->leaves[idx[i]] = values[i];
        d.push_back(idx[i]);
    }
    for (size_t j = 0; j < n_append; ++j) {
        t->leaves[n_old + j] = append[j];
        d.push_back(n_old + j);
    }
    const p252_fr* below = t->leaves;
    std::vector<p252_fr> groups, out;
    for (int l = 1; l <= t->height; ++l) {
        parents_host(d, A);
        const size_t k = d.size();
        groups.resize(k * A);
        out.resize(k);
        for (size_t i = 0; i < k; ++i) memcpy(&groups[i * A], below + d[i] * A, A * sizeof(p252_fr));
        int rc = p252_hash_batch(ctx, merkle_domain(t->arity), groups.data(), k, A, out.data(), 1, P252_MEM_HOST);
        if (rc != P252_OK) return rc;
        p252_fr* level = t->nodes + L.off[l];
        for (size_t i = 0; i < k; ++i) level[d[i]] = out[i];
        below = level;
    }
    return P252_OK;
}

}  // namespace

extern "C" {

int p252_mtree_layout(int arity, int height, uint64_t capacity, uint64_t* leaf_slots, uint64_t* node_slots,
                      uint64_t* level_offset) {
    MLayout L;
    int rc = mtree_layout(arity, height, capacity, &L);
    if (rc != P252_OK) return rc;
    if (leaf_slots) *leaf_slots = L.slots[0];
    if (node_slots) *node_slots = L.node_slots;
    if (level_offset)
        for (int l = 0; l <= height; ++l) level_offset[l] = L.off[l];
    return P252_OK;
}

int p252_mtree_build(p252_ctx* ctx, p252_mtree* tree, int flags) {
    MLayout L;
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    int rc = mtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const uint64_t n = tree->n_leaves;
    if (flags & P252_MEM_DEVICE)
        return device_done(ctx, mtree_build_device(ctx, L, tree->arity, tree->height, n, tree->leaves, tree->nodes), flags);
    // HOST: stage the leaf prefix, build on the device, copy the node slots back
    p252_fr *d_leaves = nullptr, *d_nodes = nullptr;
    auto layout = [&](Carve& c) {
        d_leaves = c.take<p252_fr>(L.slots[0]);
        d_nodes = c.take<p252_fr>(L.node_slots);
    };
    rc = with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        CU(cudaMemcpyAsync(d_leaves, tree->leaves, n * sizeof(p252_fr), cudaMemcpyHostToDevice, ctx->stream));
        const int r = mtree_build_device(ctx, L, tree->arity, tree->height, n, d_leaves, d_nodes);
        if (r != P252_OK) return r;
        CU(cudaMemcpyAsync(tree->nodes, d_nodes, L.node_slots * sizeof(p252_fr), cudaMemcpyDeviceToHost, ctx->stream));
        return P252_OK;
    });
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (rc != P252_OK) return rc;
    if (e != cudaSuccess) return fail_cuda(ctx, e, "mtree build");
    memset(tree->leaves + n, 0, (L.slots[0] - n) * sizeof(p252_fr));
    return P252_OK;
}

int p252_mtree_update(p252_ctx* ctx, p252_mtree* tree, const uint64_t* idx, const p252_fr* values, size_t n_upd,
                      const p252_fr* append, size_t n_append, size_t* n_rejected, int flags) {
    MLayout L;
    if (!ctx || (n_upd && (!idx || !values)) || (n_append && !append)) return P252_ERR_INVALID_ARGUMENT;
    int rc = mtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    if (n_upd >= 0x80000000ull || n_append >= 0x80000000ull - n_upd) return P252_ERR_INVALID_ARGUMENT;
    if (n_append > tree->capacity - tree->n_leaves) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    if (flags & P252_MEM_DEVICE) {
        if ((n_upd && (!aligned16(values) || (reinterpret_cast<uintptr_t>(idx) & 7))) || (n_append && !aligned16(append)))
            return P252_ERR_INVALID_ARGUMENT;
        if (n_upd + n_append == 0) return P252_OK;
        // keys: the leaf index, the sentinel n_new for a rejected overwrite; |D_l| <= min(batch, occupied nodes of level l)
        const int A = tree->arity, H = tree->height;
        const uint32_t T = (uint32_t)(n_upd + n_append);
        const uint64_t n_old = tree->n_leaves, n_new = n_old + n_append;
        uint64_t m[p252::kMaxDepth + 1], bound[p252::kMaxDepth + 1];
        mtree_prefix(A, H, n_new, m);
        bound[0] = T;
        for (int l = 1; l <= H; ++l) bound[l] = std::min<uint64_t>(bound[l - 1], m[l]);
        rc = tree_update_device(
            ctx, A, H, L, tree->leaves, tree->nodes, nullptr, T, sort_bits(n_new), bound, n_rejected,
            [&](uint64_t* keys, uint32_t* pos, unsigned long long* rej) {
                return p252::launch_mtree_keys(idx, (uint32_t)n_upd, n_old, T, keys, pos, rej, ctx->stream);
            },
            [&](const uint64_t* skeys, const uint32_t* spos, uint8_t* flag, uint64_t* parent) {
                return p252::launch_mtree_leaf_write(skeys, spos, T, n_new, A, values, (uint32_t)n_upd, append, tree->leaves, flag,
                                                     parent, ctx->stream);
            });
        if ((rc = device_done(ctx, rc, flags)) != P252_OK) return rc;
    } else {
        for (size_t i = 0; i < n_upd; ++i)
            if (idx[i] >= tree->n_leaves) return P252_ERR_INVALID_ARGUMENT;
        if (n_upd + n_append == 0) return P252_OK;
        rc = mtree_update_host(ctx, tree, L, idx, values, n_upd, append, n_append);
        if (rc != P252_OK) return rc;
    }
    tree->n_leaves += n_append;
    return P252_OK;
}

int p252_mtree_open_batch(p252_ctx* ctx, const p252_mtree* tree, const uint64_t* leaf_idx, size_t n, p252_fr* paths_out,
                          int flags) {
    MLayout L;
    if (!ctx || ((!leaf_idx || !paths_out) && n)) return P252_ERR_INVALID_ARGUMENT;
    int rc = mtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    const int A = tree->arity, H = tree->height;
    uint64_t m[p252::kMaxDepth + 1];
    mtree_prefix(A, H, tree->n_leaves, m);
    p252::OpenLevels lv{};
    for (int l = 0; l < H; ++l) {
        lv.off[l] = L.off[l];
        lv.m[l] = m[l];
    }
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(paths_out) || (reinterpret_cast<uintptr_t>(leaf_idx) & 7)) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        return device_done(ctx, launched(ctx, p252::launch_merkle_open(tree->leaves, tree->nodes, leaf_idx, n, A, (uint32_t)H, lv,
                                                                       paths_out, ctx->stream)), flags);
    }
    for (size_t i = 0; i < n; ++i)
        if (leaf_idx[i] >= tree->n_leaves) return P252_ERR_INVALID_ARGUMENT;
    open_host(tree->leaves, tree->nodes, leaf_idx, n, A, H, lv, paths_out);
    return P252_OK;
}

}  // extern "C"

// ---- sparse fixed-height trees (p252_smtree) -------------------------------------------------------------------
namespace {

static_assert(sizeof(size_t) == sizeof(uint64_t), "p252_smtree_len publishes its count through the size_t counter path");

int smtree_check(const p252_smtree* t, int flags, MLayout* L) {
    if (!t || t->struct_size < sizeof(p252_smtree) || !t->leaves || !t->nodes || !t->present) return P252_ERR_INVALID_ARGUMENT;
    int rc = mtree_layout(t->arity, t->height, t->capacity, L);
    if (rc != P252_OK) return rc;
    if ((flags & P252_MEM_DEVICE) && (!aligned16(t->leaves) || !aligned16(t->nodes) || (reinterpret_cast<uintptr_t>(t->present) & 3)))
        return P252_ERR_INVALID_ARGUMENT;
    return P252_OK;
}

// host-side upper bounds of |D_l|: bound[0] candidates, then at most one node per group of the level below
void smtree_bounds(const MLayout& L, int A, int H, uint64_t n0, uint64_t* bound) {
    bound[0] = n0;
    for (int l = 1; l <= H; ++l) bound[l] = std::min<uint64_t>(bound[l - 1], L.slots[l - 1] / (uint64_t)A);
}

// DEVICE build: clear every node and node presence byte, seed the climb with the leaf groups that hold a present leaf
// (k_smtree_seed also zeroes absent leaves), climb.  Only present nodes are hashed.  Temporaries: one stream-ordered
// allocation of about 17 bytes per leaf group.
int smtree_build_device(p252_ctx* ctx, const p252_smtree* t, const MLayout& L) {
    const int A = t->arity, H = t->height;
    const uint64_t G = L.slots[0] / (uint64_t)A;
    if (G >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    CU(cudaMemsetAsync(t->nodes, 0, L.node_slots * sizeof(p252_fr), ctx->stream));
    CU(cudaMemsetAsync(t->present + L.slots[0], 0, L.node_slots, ctx->stream));
    uint64_t bound[p252::kMaxDepth + 1];
    smtree_bounds(L, A, H, G, bound);
    size_t select_bytes = 0;
    CU(cub::DeviceSelect::Flagged(nullptr, select_bytes, (const uint64_t*)nullptr, (const uint8_t*)nullptr, (uint64_t*)nullptr,
                                  (int*)nullptr, (int)G, ctx->stream));
    uint64_t *parent = nullptr, *d = nullptr;
    uint8_t* flag = nullptr;
    int* cnt = nullptr;
    void* cub_tmp = nullptr;
    auto layout = [&](Carve& c) {
        parent = c.take<uint64_t>(G);
        d = c.take<uint64_t>(G);
        flag = c.take<uint8_t>(G);
        cnt = c.take<int>(H + 1);
        cub_tmp = c.take<uint8_t>(select_bytes);
    };
    return with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        const int rc = launched(ctx, p252::launch_smtree_seed(t->present, t->leaves, G, t->capacity, A, flag, parent, ctx->stream));
        if (rc != P252_OK) return rc;
        return tree_climb(ctx, A, H, L, t->leaves, t->nodes, t->present, flag, parent, d, cnt, bound, cub_tmp, select_bytes);
    });
}

// HOST update (already validated): sort and dedupe here, apply the last op per position, then per level: a dirty node
// whose children are all absent is zeroed (value and presence) without hashing, the others go through the staged
// pipeline (p252_hash_batch) and become present.
int smtree_update_host(p252_ctx* ctx, p252_smtree* t, const MLayout& L, const uint64_t* pos, const uint8_t* op,
                       const p252_fr* values, size_t n) {
    const uint64_t A = (uint64_t)t->arity;
    std::vector<uint64_t> d;
    d.reserve(n);
    for (uint32_t i : last_per_index(pos, n)) {
        const uint64_t j = pos[i];
        const bool insert = !op || op[i] == 0;
        if (insert)
            t->leaves[j] = values[i];
        else
            memset(&t->leaves[j], 0, sizeof(p252_fr));
        t->present[j] = insert ? 1 : 0;
        d.push_back(j);
    }
    const p252_fr* below = t->leaves;
    const uint8_t* below_p = t->present;
    uint8_t* node_p = t->present + L.slots[0];
    std::vector<p252_fr> groups, out;
    std::vector<uint64_t> live;
    for (int l = 1; l <= t->height; ++l) {
        parents_host(d, A);
        p252_fr* level = t->nodes + L.off[l];
        uint8_t* level_p = node_p + L.off[l];
        live.clear();
        groups.clear();
        for (uint64_t g : d) {
            bool any = false;
            for (uint64_t q = 0; q < A; ++q) any = any || below_p[g * A + q];
            if (any) {
                live.push_back(g);
                groups.insert(groups.end(), below + g * A, below + g * A + A);
            } else {
                memset(&level[g], 0, sizeof(p252_fr));
                level_p[g] = 0;
            }
        }
        out.resize(live.size());
        if (!live.empty()) {
            int rc = p252_hash_batch(ctx, merkle_domain(t->arity), groups.data(), live.size(), A, out.data(), 1, P252_MEM_HOST);
            if (rc != P252_OK) return rc;
        }
        for (size_t i = 0; i < live.size(); ++i) {
            level[live[i]] = out[i];
            level_p[live[i]] = 1;
        }
        below = level;
        below_p = level_p;
    }
    return P252_OK;
}

}  // namespace

extern "C" {

int p252_smtree_build(p252_ctx* ctx, p252_smtree* tree, int flags) {
    MLayout L;
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    int rc = smtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) return device_done(ctx, smtree_build_device(ctx, tree, L), flags);
    // HOST: stage the leaves and their presence bytes, build on the device, copy leaves, nodes and presence back
    const size_t leaf_b = L.slots[0] * sizeof(p252_fr), node_b = L.node_slots * sizeof(p252_fr);
    const size_t pres_b = L.slots[0] + L.node_slots;
    p252_smtree dt = *tree;
    auto layout = [&](Carve& c) {
        dt.leaves = c.take<p252_fr>(L.slots[0]);
        dt.nodes = c.take<p252_fr>(L.node_slots);
        dt.present = c.take<uint8_t>(pres_b);
    };
    rc = with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        CU(cudaMemcpyAsync(dt.leaves, tree->leaves, leaf_b, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(dt.present, tree->present, L.slots[0], cudaMemcpyHostToDevice, ctx->stream));
        const int r = smtree_build_device(ctx, &dt, L);
        if (r != P252_OK) return r;
        CU(cudaMemcpyAsync(tree->leaves, dt.leaves, leaf_b, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(tree->nodes, dt.nodes, node_b, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(tree->present, dt.present, pres_b, cudaMemcpyDeviceToHost, ctx->stream));
        return P252_OK;
    });
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (rc != P252_OK) return rc;
    if (e != cudaSuccess) return fail_cuda(ctx, e, "smtree build");
    return P252_OK;
}

int p252_smtree_update(p252_ctx* ctx, p252_smtree* tree, const uint64_t* pos, const uint8_t* op, const p252_fr* values,
                       size_t n, size_t* n_rejected, int flags) {
    MLayout L;
    if (!ctx || (n && (!pos || !values))) return P252_ERR_INVALID_ARGUMENT;
    int rc = smtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    if (n >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    if (flags & P252_MEM_DEVICE) {
        if (n && (!aligned16(values) || (reinterpret_cast<uintptr_t>(pos) & 7))) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        // keys: the position, the sentinel capacity for a rejected item
        const int A = tree->arity, H = tree->height;
        const uint32_t n32 = (uint32_t)n;
        uint64_t bound[p252::kMaxDepth + 1];
        smtree_bounds(L, A, H, n, bound);
        rc = tree_update_device(
            ctx, A, H, L, tree->leaves, tree->nodes, tree->present, n32, sort_bits(tree->capacity), bound, n_rejected,
            [&](uint64_t* keys, uint32_t* bpos, unsigned long long* rej) {
                return p252::launch_smtree_keys(pos, op, n32, tree->capacity, keys, bpos, rej, ctx->stream);
            },
            [&](const uint64_t* skeys, const uint32_t* sbpos, uint8_t* flag, uint64_t* parent) {
                return p252::launch_smtree_leaf_write(skeys, sbpos, n32, tree->capacity, A, op, values, tree->leaves, tree->present,
                                                      flag, parent, ctx->stream);
            });
        return device_done(ctx, rc, flags);
    }
    for (size_t i = 0; i < n; ++i)
        if (pos[i] >= tree->capacity || (op && op[i] > 1)) return P252_ERR_INVALID_ARGUMENT;
    if (n == 0) return P252_OK;
    return smtree_update_host(ctx, tree, L, pos, op, values, n);
}

int p252_smtree_len(p252_ctx* ctx, const p252_smtree* tree, uint64_t* n_present, int flags) {
    MLayout L;
    if (!ctx || !n_present) return P252_ERR_INVALID_ARGUMENT;
    int rc = smtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    *n_present = 0;
    if (flags & P252_MEM_DEVICE) {
        if ((rc = counter_begin(ctx)) != P252_OK) return rc;
        rc = launched(ctx, p252::launch_smtree_count(tree->present, tree->capacity, ctx->d_counter, ctx->stream));
        if (rc == P252_OK) rc = counter_end(ctx, reinterpret_cast<size_t*>(n_present));
        return device_done(ctx, rc, flags);
    }
    uint64_t c = 0;   // HOST: the bytes are already here
    for (uint64_t j = 0; j < tree->capacity; ++j) c += tree->present[j] != 0;
    *n_present = c;
    return P252_OK;
}

int p252_smtree_open_batch(p252_ctx* ctx, const p252_smtree* tree, const uint64_t* pos, size_t n, p252_fr* paths_out,
                           int flags) {
    MLayout L;
    if (!ctx || ((!pos || !paths_out) && n)) return P252_ERR_INVALID_ARGUMENT;
    int rc = smtree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    const int A = tree->arity, H = tree->height;
    // every slot: absent slots are already zero in memory, and so are leaf slots at or past the capacity
    p252::OpenLevels lv{};
    for (int l = 0; l < H; ++l) {
        lv.off[l] = L.off[l];
        lv.m[l] = L.slots[l];
    }
    lv.m[0] = tree->capacity;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(paths_out) || (reinterpret_cast<uintptr_t>(pos) & 7)) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        return device_done(ctx, launched(ctx, p252::launch_merkle_open(tree->leaves, tree->nodes, pos, n, A, (uint32_t)H, lv,
                                                                       paths_out, ctx->stream, tree->present)), flags);
    }
    for (size_t i = 0; i < n; ++i)
        if (pos[i] >= tree->capacity || !tree->present[pos[i]]) return P252_ERR_INVALID_ARGUMENT;
    open_host(tree->leaves, tree->nodes, pos, n, A, H, lv, paths_out);
    return P252_OK;
}

}  // extern "C"

// ---- compact sparse trees (p252_ctree) --------------------------------------------------------------------------
namespace {

struct CLayout {
    uint64_t slots[p252::kMaxDepth + 1];   // slots of level l
    uint64_t off[p252::kMaxDepth + 1];     // first slot of level l
    uint64_t total;
    uint64_t max_pos;                      // arity^height - 1
};

// slots[l] = min(max_leaves, A^(H-l)): A^(H-l) is computed only while it stays below 2^63, beyond that it exceeds any
// max_leaves
int ctree_layout(int arity, int height, uint64_t max_leaves, CLayout* L) {
    if (merkle_domain(arity) < 0 || height < 1 || height > p252::kMaxDepth) return P252_ERR_INVALID_ARGUMENT;
    if (max_leaves == 0 || max_leaves >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    const int la = arity == 4 ? 2 : 1;
    if (la * height > 64) return P252_ERR_INVALID_ARGUMENT;                // arity^height > 2^64
    uint64_t acc = 0;
    for (int l = 0; l <= height; ++l) {
        const int bits = la * (height - l);
        L->slots[l] = bits >= 63 ? max_leaves : std::min<uint64_t>(max_leaves, 1ull << bits);
        L->off[l] = acc;
        acc += L->slots[l];
    }
    L->total = acc;
    L->max_pos = la * height == 64 ? ~0ull : (1ull << (la * height)) - 1;
    return P252_OK;
}

int ctree_check(const p252_ctree* t, int flags, CLayout* L) {
    if (!t || t->struct_size < sizeof(p252_ctree) || !t->keys || !t->values || !t->count) return P252_ERR_INVALID_ARGUMENT;
    int rc = ctree_layout(t->arity, t->height, t->max_leaves, L);
    if (rc != P252_OK) return rc;
    if ((flags & P252_MEM_DEVICE) && (!aligned16(t->values) || (reinterpret_cast<uintptr_t>(t->keys) & 7) ||
                                      (reinterpret_cast<uintptr_t>(t->count) & 7)))
        return P252_ERR_INVALID_ARGUMENT;
    return P252_OK;
}

// DEVICE update, one stream, no host synchronisation, one stream-ordered allocation:
//   keys (invalid items flagged in bit 31 of the batch position) -> stable radix sort of (position, batch position)
//   over bits(arity^height) -> DeviceSelect::Flagged drops the invalid items -> the last item per position is level 0's
//   change list.  Then for l = 0..height: merge the level's change list into the level out of place (mark, two
//   exclusive scans, scatter), count, commit gated by the device flag `ok` (level 0 decides it: the new count fits
//   max_leaves), and for l < height form the next change list: the distinct parents (DeviceSelect::Flagged), their
//   dense groups gathered from the merged level, hashed by the presence-aware digest over an identity index list.
//   An empty group comes out absent, i.e. a removal.
int ctree_update_device(p252_ctx* ctx, p252_ctree* t, const CLayout& L, const uint64_t* pos, const uint8_t* op,
                        const p252_fr* values, uint32_t n, size_t* n_rejected) {
    const int A = t->arity, H = t->height, la = A == 4 ? 2 : 1;
    const uint64_t S = L.slots[0];
    uint32_t nb[p252::kMaxDepth + 1];                     // bound of level l's change list: min(n, A^(H-l))
    for (int l = 0; l <= H; ++l) nb[l] = la * (H - l) >= 32 ? n : std::min<uint32_t>(n, 1u << (la * (H - l)));
    const int end_bit = la * H;

    size_t sort_bytes = 0, select_bytes = 0, scan_bytes = 0, scan2_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                       (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, end_bit, ctx->stream));
    CU(cub::DeviceSelect::Flagged(nullptr, select_bytes, (const uint64_t*)nullptr, (const uint8_t*)nullptr, (uint64_t*)nullptr,
                                  (int*)nullptr, (int)n, ctx->stream));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)S, ctx->stream));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, scan2_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, ctx->stream));
    const size_t cub_bytes = std::max(std::max(sort_bytes, select_bytes), std::max(scan_bytes, scan2_bytes));
    uint64_t *keys, *skeys, *vkeys, *ck[2], *parent, *iota, *okeys, *stats;
    uint32_t *bpos, *sbpos, *vbpos, *kept, *K, *ins, *I, *ok;
    uint8_t *flag, *cpres, *gpres;
    p252_fr *cval, *groups, *ovals;
    int* cnt;
    void* cub_tmp;
    auto layout = [&](Carve& c) {
        keys = c.take<uint64_t>(n);
        skeys = c.take<uint64_t>(n);
        vkeys = c.take<uint64_t>(n);                       // valid items, sorted
        ck[0] = c.take<uint64_t>(n);
        ck[1] = c.take<uint64_t>(n);
        parent = c.take<uint64_t>(n);
        bpos = c.take<uint32_t>(n);
        sbpos = c.take<uint32_t>(n);
        vbpos = c.take<uint32_t>(n);
        flag = c.take<uint8_t>(n);
        cval = c.take<p252_fr>(n);                         // change values (level 0, then the digests)
        cpres = c.take<uint8_t>(n);
        groups = c.take<p252_fr>((size_t)n * A);
        gpres = c.take<uint8_t>((size_t)n * A);
        iota = c.take<uint64_t>(n);
        okeys = c.take<uint64_t>(S);                       // the merged level
        ovals = c.take<p252_fr>(S);
        kept = c.take<uint32_t>(S);
        K = c.take<uint32_t>(S);
        ins = c.take<uint32_t>(n);
        I = c.take<uint32_t>(n);
        cnt = c.take<int>(H + 3);                          // [0] valid items, [1 + l] level l's change list
        stats = c.take<uint64_t>(2);
        ok = c.take<uint32_t>(2);
        cub_tmp = c.take<uint8_t>(cub_bytes);
    };
    return with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        int rc;
        if (n_rejected && (rc = counter_begin(ctx)) != P252_OK) return rc;
        unsigned long long* rej = n_rejected ? ctx->d_counter : nullptr;
        if ((rc = launched(ctx, p252::launch_ctree_keys(pos, op, n, L.max_pos, keys, bpos, rej, ctx->stream))) != P252_OK) return rc;
        size_t b = cub_bytes;
        CU(cub::DeviceRadixSort::SortPairs(cub_tmp, b, keys, skeys, bpos, sbpos, (int)n, 0, end_bit, ctx->stream));
        if ((rc = launched(ctx, p252::launch_ctree_valid(sbpos, n, flag, ctx->stream))) != P252_OK) return rc;
        b = cub_bytes;
        CU(cub::DeviceSelect::Flagged(cub_tmp, b, skeys, flag, vkeys, cnt, (int)n, ctx->stream));
        b = cub_bytes;
        CU(cub::DeviceSelect::Flagged(cub_tmp, b, sbpos, flag, vbpos, cnt, (int)n, ctx->stream));
        if ((rc = launched(ctx, p252::launch_ctree_last(vkeys, cnt, n, flag, ctx->stream))) != P252_OK) return rc;
        b = cub_bytes;
        CU(cub::DeviceSelect::Flagged(cub_tmp, b, vkeys, flag, ck[0], cnt + 1, (int)n, ctx->stream));
        b = cub_bytes;
        CU(cub::DeviceSelect::Flagged(cub_tmp, b, vbpos, flag, bpos, cnt + 1, (int)n, ctx->stream));
        if ((rc = launched(ctx, p252::launch_ctree_leaf_changes(bpos, cnt + 1, n, op, values, cval, cpres, ctx->stream))) != P252_OK)
            return rc;
        if ((rc = launched(ctx, p252::launch_ctree_iota(iota, n, ctx->stream))) != P252_OK) return rc;
        p252_fr tag;
        p252_hash_tag(merkle_domain(A), (size_t)A, 1, &tag);
        for (int l = 0; l <= H; ++l) {
            const uint64_t s = L.slots[l];
            uint64_t* lk = t->keys + L.off[l];
            p252_fr* lv = t->values + L.off[l];
            uint64_t* lc = t->count + l;
            const uint64_t* c = ck[l & 1];
            const int* cc = cnt + 1 + l;
            if ((rc = launched(ctx, p252::launch_ctree_mark(lk, lc, s, c, cc, nb[l], cpres, kept, ins, ctx->stream))) != P252_OK)
                return rc;
            b = cub_bytes;
            CU(cub::DeviceScan::ExclusiveSum(cub_tmp, b, kept, K, (int)s, ctx->stream));
            b = cub_bytes;
            CU(cub::DeviceScan::ExclusiveSum(cub_tmp, b, ins, I, (int)nb[l], ctx->stream));
            if ((rc = launched(ctx, p252::launch_ctree_scatter(lk, lv, lc, s, c, cval, cc, nb[l], kept, K, ins, I, okeys, ovals,
                                                               ctx->stream))) != P252_OK)
                return rc;
            if ((rc = launched(ctx, p252::launch_ctree_count(lc, s, nb[l], kept, K, ins, I, l == 0, n, stats, ok, rej,
                                                             ctx->stream))) != P252_OK)
                return rc;
            if ((rc = launched(ctx, p252::launch_ctree_commit(okeys, ovals, s, stats, ok, lk, lv, lc, ctx->stream))) != P252_OK)
                return rc;
            if (l == H) break;
            // the next level's change list: distinct parents, their groups from the merged level, hashed
            if ((rc = launched(ctx, p252::launch_mtree_parents(c, cc, nb[l], A, flag, parent, ctx->stream))) != P252_OK) return rc;
            b = cub_bytes;
            CU(cub::DeviceSelect::Flagged(cub_tmp, b, parent, flag, ck[(l + 1) & 1], cnt + 2 + l, (int)nb[l], ctx->stream));
            if ((rc = launched(ctx, p252::launch_ctree_gather(okeys, ovals, stats, s, ck[(l + 1) & 1], cnt + 2 + l, nb[l + 1], A,
                                                              groups, gpres, ctx->stream))) != P252_OK)
                return rc;
            if ((rc = launched(ctx, p252::launch_mtree_digest(limbs(&tag), groups, A, cval, iota, cnt + 2 + l, nb[l + 1],
                                                              ctx->coop_max, ctx->stream, gpres, cpres))) != P252_OK)
                return rc;
        }
        return counter_end(ctx, n_rejected);
    });
}

}  // namespace

extern "C" {

int p252_ctree_layout(int arity, int height, uint64_t max_leaves, uint64_t* total_slots, uint64_t* level_offset) {
    CLayout L;
    int rc = ctree_layout(arity, height, max_leaves, &L);
    if (rc != P252_OK) return rc;
    if (total_slots) *total_slots = L.total;
    if (level_offset)
        for (int l = 0; l <= height; ++l) level_offset[l] = L.off[l];
    return P252_OK;
}

int p252_ctree_update(p252_ctx* ctx, p252_ctree* tree, const uint64_t* pos, const uint8_t* op, const p252_fr* values,
                      size_t n, size_t* n_rejected, int flags) {
    CLayout L;
    if (!ctx || (n && (!pos || !values))) return P252_ERR_INVALID_ARGUMENT;
    int rc = ctree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    if (n >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    if (flags & P252_MEM_DEVICE) {
        if (n && (!aligned16(values) || (reinterpret_cast<uintptr_t>(pos) & 7))) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        return device_done(ctx, ctree_update_device(ctx, tree, L, pos, op, values, (uint32_t)n, n_rejected), flags);
    }
    for (size_t i = 0; i < n; ++i)
        if (pos[i] > L.max_pos || (op && op[i] > 1)) return P252_ERR_INVALID_ARGUMENT;
    if (n == 0) return P252_OK;
    // HOST: stage the tree and the batch, run the device path, copy the tree back unless the batch was refused (every
    // item is valid here, so a non-zero rejection count means a capacity overflow)
    const size_t H1 = (size_t)tree->height + 1;
    const size_t kb = L.total * 8, vb = L.total * sizeof(p252_fr), cb = H1 * 8;
    p252_ctree dt = *tree;
    p252_fr* d_vals = nullptr;
    uint64_t* d_pos = nullptr;
    uint8_t* d_op = nullptr;
    auto layout = [&](Carve& c) {
        dt.values = c.take<p252_fr>(L.total);
        dt.keys = c.take<uint64_t>(L.total);
        dt.count = c.take<uint64_t>(H1);
        d_vals = c.take<p252_fr>(n);
        d_pos = c.take<uint64_t>(n);
        d_op = op ? c.take<uint8_t>(n) : nullptr;
    };
    size_t refused = 0;
    rc = with_scratch(ctx, ctx->stream, layout, [&]() -> int {
        CU(cudaMemcpyAsync(dt.values, tree->values, vb, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(dt.keys, tree->keys, kb, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(dt.count, tree->count, cb, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(d_vals, values, n * sizeof(p252_fr), cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaMemcpyAsync(d_pos, pos, n * 8, cudaMemcpyHostToDevice, ctx->stream));
        if (op) CU(cudaMemcpyAsync(d_op, op, n, cudaMemcpyHostToDevice, ctx->stream));
        const int r = ctree_update_device(ctx, &dt, L, d_pos, d_op, d_vals, (uint32_t)n, &refused);
        if (r != P252_OK) return r;
        CU(cudaStreamSynchronize(ctx->stream));   // publishes `refused`
        if (refused) return P252_OK;
        CU(cudaMemcpyAsync(tree->values, dt.values, vb, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(tree->keys, dt.keys, kb, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaMemcpyAsync(tree->count, dt.count, cb, cudaMemcpyDeviceToHost, ctx->stream));
        return P252_OK;
    });
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (rc != P252_OK) return rc;
    if (e != cudaSuccess) return fail_cuda(ctx, e, "ctree update");
    return refused ? P252_ERR_INVALID_ARGUMENT : P252_OK;
}

int p252_ctree_open_batch(p252_ctx* ctx, const p252_ctree* tree, const uint64_t* pos, size_t n, p252_fr* paths_out, int flags) {
    CLayout L;
    if (!ctx || ((!pos || !paths_out) && n)) return P252_ERR_INVALID_ARGUMENT;
    int rc = ctree_check(tree, flags, &L);
    if (rc != P252_OK) return rc;
    const int A = tree->arity, H = tree->height, la = A == 4 ? 2 : 1;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(paths_out) || (reinterpret_cast<uintptr_t>(pos) & 7)) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        p252::OpenLevels lv{};
        for (int l = 0; l < H; ++l) lv.off[l] = L.off[l];
        return device_done(ctx, launched(ctx, p252::launch_ctree_open(tree->keys, tree->values, tree->count, pos, n, A,
                                                                      (uint32_t)H, lv, paths_out, ctx->stream)), flags);
    }
    // HOST: binary searches over the sorted levels
    auto find = [&](int l, uint64_t key) -> uint64_t {   // first entry of level l whose index is >= key
        const uint64_t* k = tree->keys + L.off[l];
        return (uint64_t)(std::lower_bound(k, k + std::min(tree->count[l], L.slots[l]), key) - k);
    };
    for (size_t i = 0; i < n; ++i) {
        const uint64_t j = find(0, pos[i]);
        if (j >= std::min(tree->count[0], L.slots[0]) || tree->keys[j] != pos[i]) return P252_ERR_INVALID_ARGUMENT;
    }
    const uint64_t Az = (uint64_t)A;
    for (size_t i = 0; i < n; ++i) {
        for (int l = 0; l < H; ++l) {
            const uint64_t first = (pos[i] >> (la * l)) >> la << la;
            const uint64_t c = std::min(tree->count[l], L.slots[l]);
            const uint64_t* k = tree->keys + L.off[l];
            uint64_t j = find(l, first);
            p252_fr* dst = paths_out + (i * (size_t)H + (size_t)l) * Az;
            for (uint64_t q = 0; q < Az; ++q) {
                if (j < c && k[j] == first + q)
                    dst[q] = tree->values[L.off[l] + j++];
                else
                    memset(&dst[q], 0, sizeof(p252_fr));
            }
        }
    }
    return P252_OK;
}

}  // extern "C"

// ---- variable-length digest batches (p252_hash_batch_varlen) ----------------------------------------------------
namespace {

// The device tag table of `t` for `key` covering lengths 1..max_len: reused while it covers the call, otherwise rebuilt
// on the host (BLAKE2b stays there; fill(len, &tag) derives one tag, a failure leaves a zero tag) and uploaded on the
// context stream.  The replaced table is freed in stream order, after every kernel already enqueued that reads it; the
// pinned staging buffer is rewritten only after its previous upload has completed.
template <typename Fill>
int tag_table(p252_ctx* ctx, TagTable& t, uint64_t key, size_t max_len, Fill fill, const p252_fr** table) {
    if (t.dev && t.key == key && t.len >= max_len) {
        *table = t.dev;
        return P252_OK;
    }
    if (t.host) {
        const cudaError_t q = cudaEventQuery(t.ev);
        if (q == cudaErrorNotReady) {                      // still being read: retire it instead of waiting
            t.retired.push_back(t.host);
            t.host = nullptr;
            t.host_cap = 0;
        } else if (q != cudaSuccess) {
            return fail_cuda(ctx, q, "cudaEventQuery");
        }
    }
    if (t.host_cap < max_len + 1) {
        if (t.host) CU(cudaFreeHost(t.host));
        t.host = nullptr;
        t.host_cap = 0;
        CU(cudaHostAlloc(reinterpret_cast<void**>(&t.host), (max_len + 1) * sizeof(p252_fr), cudaHostAllocPortable));
        t.host_cap = max_len + 1;
    }
    memset(&t.host[0], 0, sizeof(p252_fr));
    for (size_t len = 1; len <= max_len; ++len)
        if (fill(len, &t.host[len]) != P252_OK) memset(&t.host[len], 0, sizeof(p252_fr));
    p252_fr* d = nullptr;
    CU(cudaMallocAsync(reinterpret_cast<void**>(&d), (max_len + 1) * sizeof(p252_fr), ctx->stream));
    cudaError_t e = cudaMemcpyAsync(d, t.host, (max_len + 1) * sizeof(p252_fr), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaEventRecord(t.ev, ctx->stream);
    if (e != cudaSuccess) {
        cudaFreeAsync(d, ctx->stream);
        return fail_cuda(ctx, e, "varlen tag table upload");
    }
    if (t.dev) CU(cudaFreeAsync(t.dev, ctx->stream));
    t.dev = d;
    t.len = max_len;
    t.key = key;
    *table = d;
    return P252_OK;
}

// Tags of Hash::digest for (domain, out_len), rebuilt only when max_len grows or (domain, out_len) changes.  Lengths the
// domain refuses (a Merkle length other than the arity) get a zero tag: k_varlen_keys rejects them before any kernel
// reads it.
int varlen_tags(p252_ctx* ctx, int domain, size_t max_len, size_t out_len, const p252_fr** table) {
    const uint64_t key = ((uint64_t)(uint32_t)domain << 32) | (uint64_t)out_len;   // out_len < 2^26
    return tag_table(ctx, ctx->vt, key, max_len, [&](size_t len, p252_fr* tag) { return p252_hash_tag(domain, len, out_len, tag); },
                     table);
}

// Tags of encrypt / decrypt (p252_encryption_tag) for message lengths 1..max_len, rebuilt only when max_len grows.
int crypt_tags(p252_ctx* ctx, size_t max_len, const p252_fr** table) {
    return tag_table(ctx, ctx->ct, 0, max_len, [](size_t len, p252_fr* tag) { return p252_encryption_tag(len, tag); }, table);
}

// One batch of n items on `st`: keys(keys, vals) writes each item's key (a length, or 0 = rejected) -> radix sort by key
// over bits(max_len) -> run(lens, perm) launches the batch kernel over the sorted order.  Temporaries are one
// stream-ordered allocation.
template <typename Keys, typename Run>
int varlen_sorted(p252_ctx* ctx, uint32_t n, uint32_t max_len, cudaStream_t st, Keys keys_launch, Run run_launch) {
    const int end_bit = sort_bits(max_len);                // keys <= max_len
    size_t sort_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                       (uint32_t*)nullptr, (int)n, 0, end_bit, st));
    uint32_t *keys = nullptr, *vals = nullptr, *lens = nullptr, *perm = nullptr;
    void* cub_tmp = nullptr;
    auto layout = [&](Carve& c) {
        keys = c.take<uint32_t>(n);
        vals = c.take<uint32_t>(n);
        lens = c.take<uint32_t>(n);
        perm = c.take<uint32_t>(n);
        cub_tmp = c.take<uint8_t>(sort_bytes);
    };
    return with_scratch(ctx, st, layout, [&]() -> int {
        const int rc = launched(ctx, keys_launch(keys, vals));
        if (rc != P252_OK) return rc;
        size_t b = sort_bytes;
        CU(cub::DeviceRadixSort::SortPairs(cub_tmp, b, keys, lens, vals, perm, (int)n, 0, end_bit, st));
        return launched(ctx, run_launch(lens, perm));
    });
}

// One digest batch on `st`: keys (length or 0 = rejected) -> radix sort by length -> the varlen digest kernel.
int varlen_run(p252_ctx* ctx, const p252_fr* tags, const p252_fr* in, uint64_t base, uint64_t n_scalars, const uint64_t* offsets,
               uint32_t n, uint32_t max_len, uint32_t fixed_len, p252_fr* out, uint32_t out_len, unsigned long long* rejected,
               cudaStream_t st) {
    return varlen_sorted(
        ctx, n, max_len, st,
        [&](uint32_t* keys, uint32_t* vals) {
            return p252::launch_varlen_keys(offsets, n, base, n_scalars, max_len, fixed_len, keys, vals, rejected, st);
        },
        [&](const uint32_t* lens, const uint32_t* perm) {
            return p252::launch_digest_varlen(tags, in, base, offsets, lens, perm, n, out, out_len, ctx->coop_max, st);
        });
}

// One encrypt / decrypt batch on `st` (see launch_crypt_varlen for the addressing; base = the value subtracted from the
// offsets to address `in`, whose length is n_scalars).
int crypt_run(p252_ctx* ctx, bool decrypt, const p252_fr* tags, const p252_fr* in, uint64_t base, uint64_t n_scalars,
              const uint64_t* offsets, uint32_t n, uint32_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* out,
              uint8_t* ok, unsigned long long* failed, unsigned long long* rejected, cudaStream_t st) {
    return varlen_sorted(
        ctx, n, max_len, st,
        [&](uint32_t* keys, uint32_t* vals) {
            return p252::launch_crypt_varlen_keys(decrypt, offsets, n, base, n_scalars, max_len, keys, vals, rejected, st);
        },
        [&](const uint32_t* lens, const uint32_t* perm) {
            return p252::launch_crypt_varlen(decrypt, tags, in, base, offsets, lens, perm, n, secret_uv, nonce, out, ok, failed,
                                             ctx->coop_max, st);
        });
}

// The chunks of a variable-length HOST batch whose offsets count elements of elem_bytes bytes (scalars, or bytes):
// consecutive item ranges of about kChunkBytesTarget input bytes (a longer item is a chunk by itself), at most
// chunk_items_max() items each; chunk k = items [bounds[k], bounds[k+1]).  out_offsets (optional, output rows of 32
// bytes): a chunk also stays within about kChunkBytesTarget output bytes.
std::vector<size_t> chunk_bounds(const uint64_t* offsets, size_t n, size_t elem_bytes,
                                 const uint64_t* out_offsets = nullptr) {
    std::vector<size_t> bounds = {0};
    for (size_t lo = 0, hi = 0; lo < n; lo = hi) {
        hi = lo + 1;
        while (hi < n && hi - lo < chunk_items_max() &&
               (offsets[hi + 1] - offsets[lo]) * elem_bytes <= kChunkBytesTarget &&
               (!out_offsets || (out_offsets[hi + 1] - out_offsets[lo]) * sizeof(p252_fr) <= kChunkBytesTarget))
            ++hi;
        bounds.push_back(hi);
    }
    return bounds;
}

// HOST batch (already validated): each chunk is staged on a slot stream -- input scalars, their offsets and the output
// rows in one stream-ordered allocation -- hashed by varlen_run with base = the chunk's first offset, and copied back.
int varlen_host(p252_ctx* ctx, const p252_fr* tags, const p252_fr* in, const uint64_t* offsets, size_t n, uint32_t max_len,
                uint32_t fixed_len, p252_fr* out, uint32_t out_len) {
    const std::vector<size_t> bounds = chunk_bounds(offsets, n, sizeof(p252_fr));
    return on_slots(ctx, false, [&](long long fail_at) -> int {
        for (size_t k = 0; k + 1 < bounds.size(); ++k) {
            const size_t lo = bounds[k], hi = bounds[k + 1], cnt = hi - lo;
            const uint64_t s0 = offsets[lo], ns = offsets[hi] - s0;
            cudaStream_t st = ctx->slots[k % kSlots].stream;
            p252_fr *d_in = nullptr, *d_out = nullptr;
            uint64_t* d_off = nullptr;
            auto layout = [&](Carve& c) {
                d_in = c.take<p252_fr>(ns);
                d_off = c.take<uint64_t>(cnt + 1);
                d_out = c.take<p252_fr>(cnt * out_len);
            };
            const int rc = with_scratch(ctx, st, layout, [&]() -> int {
                CU(cudaMemcpyAsync(d_in, in + s0, ns * sizeof(p252_fr), cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(d_off, offsets + lo, (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
                if ((long long)k == fail_at) return injected_fault(ctx);
                const int r = varlen_run(ctx, tags, d_in, s0, ns, d_off, (uint32_t)cnt, max_len, fixed_len, d_out, out_len, nullptr, st);
                if (r != P252_OK) return r;
                CU(cudaMemcpyAsync(out + lo * out_len, d_out, cnt * out_len * sizeof(p252_fr), cudaMemcpyDeviceToHost, st));
                return P252_OK;
            });
            if (rc != P252_OK) return rc;
        }
        return P252_OK;
    });
}

// HOST encrypt / decrypt batch (already validated, n > 0): each chunk is staged on a slot stream and run by crypt_run with
// base = the chunk's first offset s0.  Input, offsets, secrets, nonces, output and ok go through the slot arenas -- never
// through stream-ordered allocations -- so that join_slots(wipe) clears every secret on every exit path.
// Output of chunk [lo, hi): (ns +- cnt) scalars at out + (s0 - a0 +- lo), the chunk's part of the output CSR.
int crypt_host(p252_ctx* ctx, bool decrypt, const p252_fr* tags, const p252_fr* in, const uint64_t* offsets, size_t n,
               uint32_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* out, uint8_t* ok) {
    const std::vector<size_t> bounds = chunk_bounds(offsets, n, sizeof(p252_fr));
    p252_fr *d_in = nullptr, *d_uv = nullptr, *d_nonce = nullptr, *d_out = nullptr;
    uint64_t* d_off = nullptr;
    uint8_t* d_ok = nullptr;
    auto carve = [&](size_t k, void* arena) {              // chunk k's staging in `arena` (null: its size only)
        const size_t cnt = bounds[k + 1] - bounds[k], ns = offsets[bounds[k + 1]] - offsets[bounds[k]];
        Carve c{static_cast<uint8_t*>(arena)};
        d_in = c.take<p252_fr>(ns);
        d_off = c.take<uint64_t>(cnt + 1);
        d_uv = c.take<p252_fr>(2 * cnt);
        d_nonce = c.take<p252_fr>(cnt);
        d_out = c.take<p252_fr>(ns + cnt);                 // room for either direction
        d_ok = c.take<uint8_t>(cnt);
        return c.used;
    };
    size_t need = 0;                                       // arena bytes of the largest chunk
    for (size_t k = 0; k + 1 < bounds.size(); ++k) need = std::max(need, carve(k, nullptr));
    return on_slots(ctx, /*wipe=*/true, [&](long long fail_at) -> int {
        const uint64_t a0 = offsets[0];
        for (size_t k = 0; k + 1 < bounds.size(); ++k) {
            const size_t lo = bounds[k], hi = bounds[k + 1], cnt = hi - lo;
            const uint64_t s0 = offsets[lo], ns = offsets[hi] - s0;
            const size_t out_ns = decrypt ? ns - cnt : ns + cnt;
            const size_t out_at = decrypt ? s0 - a0 - lo : s0 - a0 + lo;
            Slot& sl = ctx->slots[k % kSlots];
            int rc = slot_reserve(ctx, sl, need, /*wipe=*/true);
            if (rc != P252_OK) return rc;
            carve(k, sl.arena);
            CU(cudaMemcpyAsync(d_in, in + s0, ns * 32, cudaMemcpyHostToDevice, sl.stream));
            CU(cudaMemcpyAsync(d_off, offsets + lo, (cnt + 1) * 8, cudaMemcpyHostToDevice, sl.stream));
            CU(cudaMemcpyAsync(d_uv, secret_uv + 2 * lo, cnt * 64, cudaMemcpyHostToDevice, sl.stream));
            CU(cudaMemcpyAsync(d_nonce, nonce + lo, cnt * 32, cudaMemcpyHostToDevice, sl.stream));
            if ((long long)k == fail_at) return injected_fault(ctx);
            rc = crypt_run(ctx, decrypt, tags, d_in, s0, ns, d_off, (uint32_t)cnt, max_len, d_uv, d_nonce, d_out,
                           decrypt ? d_ok : nullptr, nullptr, nullptr, sl.stream);
            if (rc != P252_OK) return rc;
            CU(cudaMemcpyAsync(out + out_at, d_out, out_ns * 32, cudaMemcpyDeviceToHost, sl.stream));
            if (decrypt) CU(cudaMemcpyAsync(ok + lo, d_ok, cnt, cudaMemcpyDeviceToHost, sl.stream));
        }
        return P252_OK;
    });
}

}  // namespace

extern "C" {

int p252_hash_batch_varlen(p252_ctx* ctx, int domain, const p252_fr* in, size_t n_scalars, const uint64_t* offsets, size_t n,
                           size_t max_len, p252_fr* out, size_t out_len, size_t* n_rejected, int flags) {
    bool known;
    domain_sep(domain, &known);
    if (!ctx || !known || ((!in && n_scalars) || ((!offsets || !out) && n))) return P252_ERR_INVALID_ARGUMENT;
    if (out_len == 0) return P252_ERR_INVALID_IO_PATTERN;
    const uint32_t fixed_len = domain == P252_DOMAIN_MERKLE4 ? 4u : (domain == P252_DOMAIN_MERKLE2 ? 2u : 0u);
    if (fixed_len && out_len != 1) return P252_ERR_IO_PATTERN_VIOLATION;
    if (max_len == 0 || max_len > P252_VARLEN_MAX_LEN) return P252_ERR_INVALID_ARGUMENT;
    if (n >= 0x80000000ull || out_len > 0x7fffffffull / 32) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    const p252_fr* tags = nullptr;
    int rc;
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(in) || !aligned16(out) || (reinterpret_cast<uintptr_t>(offsets) & 7)) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        if ((rc = varlen_tags(ctx, domain, max_len, out_len, &tags)) != P252_OK) return rc;
        if (n_rejected && (rc = counter_begin(ctx)) != P252_OK) return rc;
        rc = varlen_run(ctx, tags, in, 0, n_scalars, offsets, (uint32_t)n, (uint32_t)max_len, fixed_len, out, (uint32_t)out_len,
                        n_rejected ? ctx->d_counter : nullptr, ctx->stream);
        if (rc == P252_OK) rc = counter_end(ctx, n_rejected);
        return device_done(ctx, rc, flags);
    }
    // HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written
    for (size_t i = 0; i < n; ++i) {
        const uint64_t a = offsets[i], b = offsets[i + 1];
        if (a > b || b > n_scalars) return P252_ERR_INVALID_ARGUMENT;
        if (fixed_len && b - a != fixed_len) return P252_ERR_IO_PATTERN_VIOLATION;
        if (b == a) return P252_ERR_INVALID_IO_PATTERN;
        if (b - a > max_len) return P252_ERR_INVALID_ARGUMENT;
    }
    if (n == 0) return P252_OK;
    if ((rc = varlen_tags(ctx, domain, max_len, out_len, &tags)) != P252_OK) return rc;
    return varlen_host(ctx, tags, in, offsets, n, (uint32_t)max_len, fixed_len, out, (uint32_t)out_len);
}

}  // extern "C"

// ---- mixed digest batches (p252_hash_batch_mixed) --------------------------------------------------------------------
namespace {

// One mixed batch on `st`: keys (step count or 0 = rejected) with the tags derived on the device -> radix sort by step
// count -> the mixed digest kernel.  in / out hold n_scalars / n_out rows, addressed by offsets - base and
// out_offsets - obase.
int mixed_run(p252_ctx* ctx, const uint8_t* mode, const p252_fr* in, uint64_t base, uint64_t n_scalars, const uint64_t* offsets,
              const uint64_t* out_offsets, uint64_t obase, uint64_t n_out, uint32_t n, uint32_t max_len, uint32_t max_out_len,
              p252_fr* out, unsigned long long* rejected, cudaStream_t st) {
    const uint32_t max_steps = (max_len + 3) / 4 + (max_out_len + 3) / 4;
    p252_fr* tags = nullptr;
    uint2* desc = nullptr;
    auto layout = [&](Carve& c) {
        tags = c.take<p252_fr>(n);
        desc = c.take<uint2>(n);
    };
    return with_scratch(ctx, st, layout, [&]() -> int {
        return varlen_sorted(
            ctx, n, max_steps, st,
            [&](uint32_t* keys, uint32_t* vals) {
                return p252::launch_mixed_keys(mode, offsets, base, n_scalars, out_offsets, obase, n_out, n, max_len, max_out_len,
                                               out, keys, vals, tags, desc, rejected, st);
            },
            [&](const uint32_t*, const uint32_t* perm) {
                return p252::launch_digest_mixed(tags, desc, in, base, offsets, obase, out_offsets, perm, n, out, ctx->coop_max,
                                                 st);
            });
    });
}

// HOST batch (already validated, so both offset arrays are non-decreasing): as varlen_host, with chunks bounded by input
// and output bytes; each chunk stages its modes, both offset slices and its input rows, and copies back its output rows.
int mixed_host(p252_ctx* ctx, const uint8_t* mode, const p252_fr* in, const uint64_t* offsets, const uint64_t* out_offsets,
               size_t n, uint32_t max_len, uint32_t max_out_len, p252_fr* out) {
    const std::vector<size_t> bounds = chunk_bounds(offsets, n, sizeof(p252_fr), out_offsets);
    return on_slots(ctx, false, [&](long long fail_at) -> int {
        for (size_t k = 0; k + 1 < bounds.size(); ++k) {
            const size_t lo = bounds[k], hi = bounds[k + 1], cnt = hi - lo;
            const uint64_t s0 = offsets[lo], ns = offsets[hi] - s0, o0 = out_offsets[lo], no = out_offsets[hi] - o0;
            cudaStream_t st = ctx->slots[k % kSlots].stream;
            p252_fr *d_in = nullptr, *d_out = nullptr;
            uint64_t *d_off = nullptr, *d_ooff = nullptr;
            uint8_t* d_mode = nullptr;
            auto layout = [&](Carve& c) {
                d_in = c.take<p252_fr>(ns);
                d_off = c.take<uint64_t>(cnt + 1);
                d_ooff = c.take<uint64_t>(cnt + 1);
                d_mode = c.take<uint8_t>(cnt);
                d_out = c.take<p252_fr>(no);
            };
            const int rc = with_scratch(ctx, st, layout, [&]() -> int {
                CU(cudaMemcpyAsync(d_in, in + s0, ns * sizeof(p252_fr), cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(d_off, offsets + lo, (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(d_ooff, out_offsets + lo, (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(d_mode, mode + lo, cnt, cudaMemcpyHostToDevice, st));
                if ((long long)k == fail_at) return injected_fault(ctx);
                const int r = mixed_run(ctx, d_mode, d_in, s0, ns, d_off, d_ooff, o0, no, (uint32_t)cnt, max_len, max_out_len,
                                        d_out, nullptr, st);
                if (r != P252_OK) return r;
                CU(cudaMemcpyAsync(out + o0, d_out, no * sizeof(p252_fr), cudaMemcpyDeviceToHost, st));
                return P252_OK;
            });
            if (rc != P252_OK) return rc;
        }
        return P252_OK;
    });
}

// The status of item i of a HOST mixed batch, in the order of the header's item checks
int mixed_item_status(const uint8_t* mode, const uint64_t* offsets, const uint64_t* out_offsets, size_t i, size_t n_scalars,
                      size_t n_out, size_t max_len, size_t max_out_len) {
    const uint64_t a = offsets[i], b = offsets[i + 1], oa = out_offsets[i], ob = out_offsets[i + 1];
    if (mode[i] & ~(P252_MIXED_TRUNCATED | 3)) return P252_ERR_INVALID_ARGUMENT;   // domain bits and truncation only
    if (a > b || b > n_scalars) return P252_ERR_INVALID_ARGUMENT;
    if (oa > ob || ob > n_out) return P252_ERR_INVALID_ARGUMENT;
    const int domain = mode[i] & 3;
    const uint64_t arity = domain == P252_DOMAIN_MERKLE4 ? 4 : (domain == P252_DOMAIN_MERKLE2 ? 2 : 0);
    if (arity && (b - a != arity || ob - oa != 1)) return P252_ERR_IO_PATTERN_VIOLATION;
    if (b == a || ob == oa) return P252_ERR_INVALID_IO_PATTERN;
    if (b - a > max_len || ob - oa > max_out_len) return P252_ERR_INVALID_ARGUMENT;
    return P252_OK;
}

}  // namespace

extern "C" {

int p252_hash_batch_mixed(p252_ctx* ctx, const uint8_t* mode, const p252_fr* in, size_t n_scalars, const uint64_t* offsets,
                          size_t n, size_t max_len, p252_fr* out, size_t n_out, const uint64_t* out_offsets, size_t max_out_len,
                          size_t* n_rejected, int flags) {
    if (!ctx || (!in && n_scalars) || (!out && n_out) || ((!mode || !offsets || !out_offsets || !out) && n))
        return P252_ERR_INVALID_ARGUMENT;
    if (n >= 0x80000000ull || max_len == 0 || max_len > P252_VARLEN_MAX_LEN || max_out_len == 0 ||
        max_out_len > P252_VARLEN_MAX_LEN)
        return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    int rc;
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(in) || !aligned16(out) || (reinterpret_cast<uintptr_t>(offsets) & 7) ||
            (reinterpret_cast<uintptr_t>(out_offsets) & 7))
            return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        if (n_rejected && (rc = counter_begin(ctx)) != P252_OK) return rc;
        rc = mixed_run(ctx, mode, in, 0, n_scalars, offsets, out_offsets, 0, n_out, (uint32_t)n, (uint32_t)max_len,
                       (uint32_t)max_out_len, out, n_rejected ? ctx->d_counter : nullptr, ctx->stream);
        if (rc == P252_OK) rc = counter_end(ctx, n_rejected);
        return device_done(ctx, rc, flags);
    }
    // HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written
    for (size_t i = 0; i < n; ++i)
        if ((rc = mixed_item_status(mode, offsets, out_offsets, i, n_scalars, n_out, max_len, max_out_len)) != P252_OK) return rc;
    if (n == 0) return P252_OK;
    return mixed_host(ctx, mode, in, offsets, out_offsets, n, (uint32_t)max_len, (uint32_t)max_out_len, out);
}

}  // extern "C"

// ---- variable-length encrypt / decrypt batches (p252_encrypt_batch_varlen / p252_decrypt_batch_varlen) ----------------
namespace {

int crypt_varlen(p252_ctx* ctx, bool decrypt, const p252_fr* in, size_t n_scalars, const uint64_t* offsets, size_t n,
                 size_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* out, uint8_t* ok, size_t* n_failed,
                 size_t* n_rejected, int flags) {
    if (!ctx || ((!in || !offsets || !secret_uv || !nonce || !out || (decrypt && !ok)) && n)) return P252_ERR_INVALID_ARGUMENT;
    if (max_len == 0 || max_len > P252_VARLEN_MAX_LEN || n >= 0x80000000ull) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_failed) *n_failed = 0;
    if (n_rejected) *n_rejected = 0;
    const p252_fr* tags = nullptr;
    int rc;
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(in) || !aligned16(secret_uv) || !aligned16(nonce) || !aligned16(out) ||
            (reinterpret_cast<uintptr_t>(offsets) & 7))
            return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        if ((rc = crypt_tags(ctx, max_len, &tags)) != P252_OK) return rc;
        // counter slot 0: authentication failures (decrypt), slot 1: rejected items
        if ((n_failed || n_rejected) && (rc = counter_begin(ctx, p252_ctx::kCounters)) != P252_OK) return rc;
        rc = crypt_run(ctx, decrypt, tags, in, 0, n_scalars, offsets, (uint32_t)n, (uint32_t)max_len, secret_uv, nonce, out, ok,
                       n_failed ? ctx->d_counter : nullptr, n_rejected ? ctx->d_counter + 1 : nullptr, ctx->stream);
        if (rc == P252_OK) rc = counter_end(ctx, n_failed, 0);
        if (rc == P252_OK) rc = counter_end(ctx, n_rejected, 1);
        return device_done(ctx, rc, flags);
    }
    // HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written.
    // With every item valid the output ranges are disjoint and inside the output, so the decrypt range conditions of the
    // device path need no check here.
    const uint64_t kMin = decrypt ? 2 : 1;
    for (size_t i = 0; i < n; ++i) {
        const uint64_t a = offsets[i], b = offsets[i + 1];
        if (a < offsets[0] || a > b || b > offsets[n] || offsets[n] > n_scalars) return P252_ERR_INVALID_ARGUMENT;
        if (b - a < kMin) return P252_ERR_INVALID_IO_PATTERN;                 // as p252_encryption_tag(0)
        if (b - a > max_len + kMin - 1) return P252_ERR_INVALID_ARGUMENT;
    }
    if (n == 0) return P252_OK;
    if ((rc = crypt_tags(ctx, max_len, &tags)) != P252_OK) return rc;
    rc = crypt_host(ctx, decrypt, tags, in, offsets, n, (uint32_t)max_len, secret_uv, nonce, out, ok);
    if (rc == P252_OK && n_failed) *n_failed = count_zero(ok, n);
    return rc;
}

}  // namespace

extern "C" {

int p252_encrypt_batch_varlen(p252_ctx* ctx, const p252_fr* msg, size_t n_scalars, const uint64_t* offsets, size_t n,
                              size_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* cipher,
                              size_t* n_rejected, int flags) {
    return crypt_varlen(ctx, false, msg, n_scalars, offsets, n, max_len, secret_uv, nonce, cipher, nullptr, nullptr, n_rejected,
                        flags);
}

int p252_decrypt_batch_varlen(p252_ctx* ctx, const p252_fr* cipher, size_t n_scalars, const uint64_t* offsets, size_t n,
                              size_t max_len, const p252_fr* secret_uv, const p252_fr* nonce, p252_fr* msg, uint8_t* ok,
                              size_t* n_failed, size_t* n_rejected, int flags) {
    return crypt_varlen(ctx, true, cipher, n_scalars, offsets, n, max_len, secret_uv, nonce, msg, ok, n_failed, n_rejected,
                        flags);
}

}  // extern "C"

// ---- BlsScalar::hash_to_scalar batches (p252_hash_to_scalar_batch) ---------------------------------------------------
namespace {

// One batch on `st` (item i = bytes[offsets[i] - base ..) of n_bytes): with max_len <= 128 every item is one block and
// k_hash_to_scalar runs in input order, counting rejected items itself; otherwise items are sorted by block count first
// (varlen_sorted, which counts them in the keys kernel).
int hash_to_scalar_run(p252_ctx* ctx, const uint8_t* bytes, uint64_t base, uint64_t n_bytes, const uint64_t* offsets, uint32_t n,
                       uint32_t max_len, p252_fr* out, unsigned long long* rejected, cudaStream_t st) {
    if (max_len <= 128)
        return launched(ctx, p252::launch_hash_to_scalar(bytes, base, n_bytes, offsets, nullptr, n, max_len, out,
                                                         rejected, st));
    const uint32_t max_blocks = (max_len + 127) / 128;
    return varlen_sorted(
        ctx, n, max_blocks, st,
        [&](uint32_t* keys, uint32_t* vals) {
            return p252::launch_hash_to_scalar_keys(offsets, n, base, n_bytes, max_len, keys, vals, rejected, st);
        },
        [&](const uint32_t*, const uint32_t* perm) {
            return p252::launch_hash_to_scalar(bytes, base, n_bytes, offsets, perm, n, max_len, out, nullptr, st);
        });
}

// HOST batch (already validated): as varlen_host, with chunks of about kChunkBytesTarget message bytes
int hash_to_scalar_host(p252_ctx* ctx, const uint8_t* bytes, const uint64_t* offsets, size_t n, uint32_t max_len, p252_fr* out) {
    const std::vector<size_t> bounds = chunk_bounds(offsets, n, 1);
    return on_slots(ctx, false, [&](long long fail_at) -> int {
        for (size_t k = 0; k + 1 < bounds.size(); ++k) {
            const size_t lo = bounds[k], hi = bounds[k + 1], cnt = hi - lo;
            const uint64_t s0 = offsets[lo], nb = offsets[hi] - s0;
            cudaStream_t st = ctx->slots[k % kSlots].stream;
            uint8_t* d_in = nullptr;
            uint64_t* d_off = nullptr;
            p252_fr* d_out = nullptr;
            auto layout = [&](Carve& c) {
                d_in = c.take<uint8_t>(nb);
                d_off = c.take<uint64_t>(cnt + 1);
                d_out = c.take<p252_fr>(cnt);
            };
            const int rc = with_scratch(ctx, st, layout, [&]() -> int {
                if (nb) CU(cudaMemcpyAsync(d_in, bytes + s0, nb, cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(d_off, offsets + lo, (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
                if ((long long)k == fail_at) return injected_fault(ctx);
                const int r = hash_to_scalar_run(ctx, d_in, s0, nb, d_off, (uint32_t)cnt, max_len, d_out, nullptr, st);
                if (r != P252_OK) return r;
                CU(cudaMemcpyAsync(out + lo, d_out, cnt * sizeof(p252_fr), cudaMemcpyDeviceToHost, st));
                return P252_OK;
            });
            if (rc != P252_OK) return rc;
        }
        return P252_OK;
    });
}

}  // namespace

extern "C" {

int p252_hash_to_scalar_batch(p252_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const uint64_t* offsets, size_t n,
                              size_t max_len, p252_fr* out, size_t* n_rejected, int flags) {
    if (!ctx || (!bytes && n_bytes) || ((!offsets || !out) && n)) return P252_ERR_INVALID_ARGUMENT;
    if (n >= 0x80000000ull || max_len > P252_HASH_TO_SCALAR_MAX_LEN) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (n_rejected) *n_rejected = 0;
    int rc;
    if (flags & P252_MEM_DEVICE) {
        if (!aligned16(out) || (reinterpret_cast<uintptr_t>(offsets) & 7)) return P252_ERR_INVALID_ARGUMENT;
        if (n == 0) return P252_OK;
        if (n_rejected && (rc = counter_begin(ctx)) != P252_OK) return rc;
        rc = hash_to_scalar_run(ctx, bytes, 0, n_bytes, offsets, (uint32_t)n, (uint32_t)max_len, out,
                                n_rejected ? ctx->d_counter : nullptr, ctx->stream);
        if (rc == P252_OK) rc = counter_end(ctx, n_rejected);
        return device_done(ctx, rc, flags);
    }
    // HOST: the whole batch is checked first; the lowest-index invalid item decides the status and nothing is written
    for (size_t i = 0; i < n; ++i) {
        const uint64_t a = offsets[i], b = offsets[i + 1];
        if (a > b || b > n_bytes || b - a > max_len) return P252_ERR_INVALID_ARGUMENT;
    }
    if (n == 0) return P252_OK;
    return hash_to_scalar_host(ctx, bytes, offsets, n, (uint32_t)max_len, out);
}

}  // extern "C"

extern "C" {

// ---- multi-GPU ------------------------------------------------------------------------------------------
int p252_dist_unique_id(uint8_t id[P252_NCCL_UNIQUE_ID_BYTES]) {
    static_assert(sizeof(ncclUniqueId) <= P252_NCCL_UNIQUE_ID_BYTES, "unique id size");
    p252_ctx* ctx = nullptr;
    if (!id) return P252_ERR_INVALID_ARGUMENT;
    if (!nccl().ok) return fail_nccl(ctx, ncclSystemError, "dlopen(libnccl.so.2)");
    ncclUniqueId u;
    NC(nccl().GetUniqueId(&u));
    memset(id, 0, P252_NCCL_UNIQUE_ID_BYTES);
    memcpy(id, &u, sizeof u);
    return P252_OK;
}

int p252_dist_init(p252_ctx* ctx, const uint8_t id[P252_NCCL_UNIQUE_ID_BYTES], int rank, int nranks) {
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return P252_ERR_INVALID_ARGUMENT;
    if (ctx->comm) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (!nccl().ok) return fail_nccl(ctx, ncclSystemError, "dlopen(libnccl.so.2)");
    ncclUniqueId u;
    memcpy(&u, id, sizeof u);
    NC(nccl().CommInitRank(&ctx->comm, nranks, u, rank));
    ctx->rank = rank;
    ctx->nranks = nranks;
    CU(cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
    return P252_OK;
}

int p252_dist_finalize(p252_ctx* ctx) {
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    if (ctx->comm) {
        CU(cudaStreamSynchronize(ctx->comm_stream));
        NC(nccl().CommDestroy(ctx->comm));
        ctx->comm = nullptr;
    }
    if (ctx->comm_stream) {
        cudaStreamDestroy(ctx->comm_stream);
        ctx->comm_stream = nullptr;
    }
    ctx->rank = 0;
    ctx->nranks = 1;
    return P252_OK;
}

// Contiguous sharding: rank r owns nodes [r*M/G, (r+1)*M/G) of every level with M % G == 0 nodes, whose
// children are exactly rank r's slice of the level below -- so the compute stream climbs its own
// subtree without waiting, while the all-gather of each finished level (the level's replication to
// all GPUs over NVLink) runs on a second stream.  Smaller levels are computed redundantly by every
// rank from the gathered level below.
int p252_merkle4_shard_plan(size_t n_leaves_total, int nranks, int rank, p252_level_plan* levels, int capacity,
                            int* n_levels) {
    if (nranks < 1 || rank < 0 || rank >= nranks) return P252_ERR_INVALID_ARGUMENT;
    int lv = 0;
    int rc = p252_merkle4_tree_nodes(n_leaves_total, nullptr, &lv);
    if (rc != P252_OK) return rc;
    if (n_leaves_total % (size_t)nranks || (n_leaves_total / nranks) % 4) return P252_ERR_INVALID_ARGUMENT;
    if (n_levels) *n_levels = lv;
    if (!levels) return P252_OK;
    if (capacity < lv) return P252_ERR_INVALID_ARGUMENT;
    uint64_t off = 0, m = n_leaves_total / 4;
    for (int l = 0; l < lv; ++l, m /= 4) {
        p252_level_plan& p = levels[l];
        p.level_offset = off;
        p.level_size = m;
        p.sharded = (m % (uint64_t)nranks == 0) ? 1 : 0;
        p.my_count = p.sharded ? m / nranks : m;
        p.my_offset = p.sharded ? (uint64_t)rank * p.my_count : 0;
        p.reserved = 0;
        off += m;
    }
    return P252_OK;
}

int p252_merkle4_build_dist(p252_ctx* ctx, const p252_fr* leaves_shard, size_t n_leaves_total, p252_fr* nodes_out,
                            int flags) {
    if (!ctx || !leaves_shard || !nodes_out) return P252_ERR_INVALID_ARGUMENT;
    if (!(flags & P252_MEM_DEVICE)) return P252_ERR_INVALID_ARGUMENT;   // shards live on the GPU
    if (!aligned16(leaves_shard) || !aligned16(nodes_out)) return P252_ERR_INVALID_ARGUMENT;
    const int G = ctx->nranks, r = ctx->rank;
    if (G > 1 && !ctx->comm) return P252_ERR_INVALID_ARGUMENT;
    p252_level_plan plan[64];
    int lv = 0;
    int rc = p252_merkle4_shard_plan(n_leaves_total, G, r, plan, 64, &lv);
    if (rc != P252_OK) return rc;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    p252_fr tag;
    p252_hash_tag(P252_DOMAIN_MERKLE4, 4, 1, &tag);

    const bool timing = (flags & P252_TIMING) != 0;
    const bool no_gather = (flags & P252_NO_GATHER) != 0;
    if (timing) {
        // events with timing enabled, created once per context and reused
        while ((int)ctx->level_events.size() < lv) {
            p252_ctx::LevelEvents le;
            for (cudaEvent_t* ev : {&le.k0, &le.k1, &le.g0, &le.g1}) CU(cudaEventCreate(ev));
            ctx->level_events.push_back(le);
        }
        ctx->level_info.assign((size_t)lv, p252_level_timing{});
        ctx->level_gathered.assign((size_t)lv, 0);
    }
    ctx->timed_levels = timing ? lv : 0;

    const p252_fr* below_full = nullptr;        // complete level below (valid once gathered)
    const p252_fr* below_mine = leaves_shard;   // this rank's slice of the level below
    bool gather_in_flight = false;
    CU(cudaEventRecord(ctx->ev_comm, ctx->stream));
    for (int l = 0; l < lv; ++l) {
        const p252_level_plan& p = plan[l];
        p252_fr* level = nodes_out + p.level_offset;
        if (timing) {
            ctx->level_info[(size_t)l].nodes = p.level_size;
            ctx->level_info[(size_t)l].my_nodes = p.my_count;
        }
        if (p.sharded) {
            // the first level is always sharded (n_leaves_total / G is a multiple of 4)
            if (timing) CU(cudaEventRecord(ctx->level_events[(size_t)l].k0, ctx->stream));
            rc = launched(ctx, p252::launch_digest(limbs(&tag), below_mine, p.my_count, 4, level + p.my_offset, 1, false,
                                                   ctx->coop_max, ctx->stream));
            if (rc != P252_OK) return rc;
            if (timing) CU(cudaEventRecord(ctx->level_events[(size_t)l].k1, ctx->stream));
            if (G > 1 && !no_gather) {
                CU(cudaEventRecord(ctx->ev_level, ctx->stream));
                CU(cudaStreamWaitEvent(ctx->comm_stream, ctx->ev_level, 0));
                if (timing) CU(cudaEventRecord(ctx->level_events[(size_t)l].g0, ctx->comm_stream));
                NC(nccl().AllGather(level + p.my_offset, level, p.my_count * 4, ncclUint64, ctx->comm, ctx->comm_stream));
                if (timing) {
                    CU(cudaEventRecord(ctx->level_events[(size_t)l].g1, ctx->comm_stream));
                    ctx->level_gathered[(size_t)l] = 1;
                    ctx->level_info[(size_t)l].gather_bytes = p.level_size * sizeof(p252_fr);
                }
                CU(cudaEventRecord(ctx->ev_comm, ctx->comm_stream));
                gather_in_flight = true;
            }
            below_mine = level + p.my_offset;
        } else {
            if (gather_in_flight) {   // needs the complete level below on this rank
                CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_comm, 0));
                gather_in_flight = false;
            }
            if (timing) CU(cudaEventRecord(ctx->level_events[(size_t)l].k0, ctx->stream));
            rc = launched(ctx, p252::launch_digest(limbs(&tag), below_full, p.level_size, 4, level, 1, false, ctx->coop_max,
                                                   ctx->stream));
            if (rc != P252_OK) return rc;
            if (timing) CU(cudaEventRecord(ctx->level_events[(size_t)l].k1, ctx->stream));
        }
        below_full = level;
    }
    // every level must be complete on every rank before the call is considered done
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_comm, 0));
    if (timing) CU(cudaEventRecord(ctx->ev_tree_end, ctx->stream));
    return device_done(ctx, P252_OK, flags);
}

int p252_tree_level_timings(p252_ctx* ctx, p252_level_timing* levels, int capacity, int* n_levels, float* total_ms) {
    if (!ctx) return P252_ERR_INVALID_ARGUMENT;
    P252_LOCK(ctx);
    DeviceGuard g(ctx->device);
    const int lv = ctx->timed_levels;
    if (n_levels) *n_levels = lv;
    if (lv == 0) return P252_ERR_INVALID_ARGUMENT;   // no P252_TIMING build on this context yet
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->comm_stream) CU(cudaStreamSynchronize(ctx->comm_stream));
    if (total_ms) CU(cudaEventElapsedTime(total_ms, ctx->level_events[0].k0, ctx->ev_tree_end));
    if (!levels) return P252_OK;
    if (capacity < lv) return P252_ERR_INVALID_ARGUMENT;
    for (int l = 0; l < lv; ++l) {
        p252_level_timing t = ctx->level_info[(size_t)l];
        CU(cudaEventElapsedTime(&t.kernel_ms, ctx->level_events[(size_t)l].k0, ctx->level_events[(size_t)l].k1));
        t.gather_ms = 0.f;
        if (ctx->level_gathered[(size_t)l])
            CU(cudaEventElapsedTime(&t.gather_ms, ctx->level_events[(size_t)l].g0, ctx->level_events[(size_t)l].g1));
        levels[l] = t;
    }
    return P252_OK;
}

}  // extern "C"
