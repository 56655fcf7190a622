// b2_api.cu — the C ABI (include/b2rpc.h) over the sm_90a kernels.
// Host code is plain C++ + the CUDA runtime; nothing here computes on the CPU:
// without a CUDA device every entry point fails with B2_E_NO_DEVICE.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdio.h>
#include <time.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>
#include "b2_kernels.cuh"
#include "b2_h2.cuh"

using namespace b2;

static thread_local char g_err[512] = "";
static void set_err(const char* fmt, const char* a = "", const char* b = "") { snprintf(g_err, sizeof g_err, fmt, a, b); }

#define CU(call)                                                                          \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess) { set_err("%s: %s", #call, cudaGetErrorString(e_)); return B2_E_CUDA; } \
    } while (0)

namespace {
constexpr int kMaxStages = 16;
constexpr uint32_t kSmallBytes = 128 << 10;        // batches up to this size take the latency path
constexpr uint32_t kSmallRuns = 512, kSmallMsgs = 1024;   // == kSmallThreads, 2 * kSmallThreads of k_small
constexpr size_t kSmallBlock = 64 + kSmallRuns * 32 + kSmallMsgs * (64 + 16) + (kSmallBytes + kSmallMsgs * 80 + 4096);
// the compact output block of a small batch, as k_small and k_ring write it: [totals 64 | run statuses | msgs | refs | resp]
// (msgs is bounded by max_msgs too: d_frame_off / d_aux / d_jobs / d_heads ... are sized by it)
struct SmallLayout { uint32_t msgs, resp, off_rs, off_msgs, off_refs, off_resp, total; };
SmallLayout small_layout(uint32_t nbytes, uint32_t n_runs, uint32_t max_msgs) {
    const uint32_t mb = std::min(std::min(nbytes / 12 + 1, kSmallMsgs), max_msgs), resp = nbytes + mb * 80 + 2048, off_msgs = 64 + n_runs * 32;
    const uint32_t off_refs = off_msgs + mb * 64, off_resp = (off_refs + mb * 16 + 255u) & ~255u;
    return { mb, resp, 64, off_msgs, off_refs, off_resp, off_resp + resp };
}
// a ring slot's stream section (b2_stream_ring_enable), and the device staging k_ring fills before it pushes the section:
// [counters 64 | events | msgs | ctrl | run_ctrl | out], each part sized for what one ticket of <= kSmallMsgs messages can produce
// (touched streams <= messages; per message at most one RST frame, per stream one FEEDBACK and one CLOSE frame)
constexpr uint32_t kSecEvents = 64, kSecMsgs = kSecEvents + kSmallMsgs * 80, kSecCtrl = kSecMsgs + kSmallMsgs * 32,
                   kSecRunCtrl = kSecCtrl + 3 * kStreamCtrlMax * kSmallMsgs, kSecOut = kSecRunCtrl + kSmallRuns * 8;
struct Stage { const char* name; cudaEvent_t ev; };
// Which resident kernel a context's ring runs, fixed by its first ring call: k_ring (b2_ring_start / b2_ring_submit), k_ring with the
// stream pass (b2_stream_ring_enable), k_ring<RingBody::stream_writes> with the stream pass and the write pass (b2_stream_ring_write_enable),
// k_ring<RingBody::requests> with the request phase (b2_client_ring_enable), k_ring<RingBody::replies> with the reply phase
// (b2_ring_turn_enable), k_h2_ring (b2_h2_ring_enable) or k_h2_client_ring (b2_h2_client_ring_enable)
enum class RingKind { none, batch, batch_streams, batch_stream_writes, batch_client, batch_replies, h2_server, h2_client };
// The kinds whose tickets pack records after the runs (k_ring<RingBody::requests> / <RingBody::replies>)
bool ring_packs(RingKind k) { return k == RingKind::batch_client || k == RingKind::batch_replies; }
// The kinds whose tickets run the stream pass: the table belongs to an outstanding ticket, tickets are collected in ticket order, the
// kernel parks behind a ticket that overflows the compact block, and the slot carries a stream section
bool ring_runs_streams(RingKind k) { return k == RingKind::batch_streams || k == RingKind::batch_stream_writes; }
// A slot's layout: the header (RingSlotHdr, then the kind's per-ticket args) in the first 256 bytes, then each part 256-byte aligned
struct SlotLayout {
    uint64_t end = 256;
    uint32_t add(uint64_t bytes) { const uint64_t off = end; end = (end + bytes + 255u) & ~255ull; return (uint32_t)off; }
};
}

// The kernels of a fused pass in b2_resident_plan's order: k_fused, then the ones launched between two k_fused passes (DESIGN §3)
enum : int { kPlanFused, kPlanSearch, kPlanWalk, kPlanResolve, kPlanSlow, kPlanKernels };
struct b2_ctx {
    b2_options opt;
    DevConfig cfg;
    std::vector<DevMethod> methods;
    // device
    uint8_t* d_bytes = nullptr; b2_run* d_runs = nullptr; uint32_t* d_run_tile_base = nullptr;
    TileRec* d_tiles = nullptr; uint32_t* d_tile_base = nullptr; uint32_t* d_tile_scratch = nullptr; TileRec* d_head_recs = nullptr; uint32_t* d_tile_spec = nullptr; b2_run_status* d_run_status = nullptr;
    uint32_t* d_frame_off = nullptr; uint32_t* d_frame_run = nullptr; b2_msg_desc* d_msgs = nullptr; MsgAux* d_aux = nullptr; PackJob* d_jobs = nullptr; uint32_t* d_slow_idx = nullptr; uint8_t* d_heads = nullptr;
    uint32_t* d_slot = nullptr; uint32_t* d_scan_tmp = nullptr; uint8_t* d_resp = nullptr; uint8_t* d_unz = nullptr; uint16_t* d_snappy_tab = nullptr; HpackState* d_hpack = nullptr; H2Conn* d_h2 = nullptr; H2Stream* d_h2_streams = nullptr; uint8_t* d_h2_slots = nullptr; uint32_t h2_max_conns = B2_H2_MAX_CONNS, h2_pending = B2_H2_MAX_PENDING, h2_stream_bytes = B2_H2_STREAM_BYTES; uint64_t h2_last_in = 0, h2_last_out = 0;   // sizes of the last h2 batch still on the device
    uint32_t* d_frame_row = nullptr; uint4* d_rows = nullptr;
    std::vector<uint8_t> h2_gunzip; uint8_t* d_h2_gz_merge = nullptr;     // host mirror of the kH2Gunzip bits; merge scratch, B2_H2_HEADER_BYTES per run
    // persistent latency kernel (b2_ring_*): pinned + mapped submit ring, its own stream.  ring_slots: allocated (by the first ring call
    // that needs them); the slot parts of each kind live in that kind's kernel arguments (ring_dev: runs, staged input, output, stream section)
    RingKind ring_kind = RingKind::none; RingDev ring_dev = {}; PackRingDev pr_dev = {}; H2RingDev h2r_dev = {}; H2ClientRingDev h2c_dev = {};
    uint8_t* ring_slots = nullptr; volatile uint32_t* ring_ctl = nullptr; uint32_t* d_ring_ticket = nullptr; cudaStream_t ring_stream = nullptr;
    uint32_t ring_next = 1, ring_stride = 0; bool ring_collected[8] = { true, true, true, true, true, true, true, true };
    const void* ring_bytes[8] = {}; const void* ring_pin_base = nullptr; unsigned long long ring_pin_dev = 0; uint64_t ring_launches = 0;
    // the stream pass on the ring (batch_streams): the ring's StreamPass writes its results into d_st_ring, k_ring pushes them to the
    // slot's section; tickets are collected in order (ring_next_wait); st_view_ticket: the ticket b2_stream_results describes (0: the last
    // batch call's pass)
    StreamPass sp_ring = {}; uint8_t* d_st_ring = nullptr; uint32_t ring_next_wait = 1, st_view_ticket = 0;
    // the caps every ticket of an h2 ring (k_h2_ring, k_h2_client_ring) is served with
    uint32_t h2r_max_bytes = 0, h2r_msg_cap = 0, h2r_out_cap = 0, h2r_replies_cap = 0;
    uint32_t h2r_max_resps = 0, h2r_resp_out_cap = 0; H2TurnDev h2t_dev = {};   // ... and the host replies of a turn (b2_h2_ring_turn_enable)
    uint32_t h2c_max_bytes = 0, h2c_call_cap = 0, h2c_out_cap = 0, h2c_max_reqs = 0, h2c_req_out_cap = 0;
    uint32_t pr_max_bytes = 0, pr_max_recs = 0, pr_out_cap = 0;            // ... and of the client ring or the turn ring (ring_packs)
    // the stream write ring (k_ring<RingBody::stream_writes>): its caps, its slot parts and the write pass's device scratch (d_swr)
    uint32_t swr_max_bytes = 0, swr_max_writes = 0, swr_out_cap = 0; SwRingDev swr_dev = {}; uint8_t* d_swr = nullptr;
    ulonglong2* d_iov = nullptr; b2_iovec* h_iov = nullptr; const void* host_bytes = nullptr;      // B2_RESP_IOVEC
    uint4* d_refs = nullptr; b2_resp_ref* h_refs = nullptr; int input_mode = B2_INPUT_COPY, resp_mode = B2_RESP_COPY; const uint8_t* pull_bytes = nullptr;
    uint32_t* d_crc_adv = nullptr; unsigned long long* d_counters = nullptr; uint32_t* d_totals = nullptr; DevMethod* d_methods = nullptr;
    size_t meta_tile_off = 0; uint32_t max_tiles = 0; uint32_t n_sms = 132; bool use_tma_pack = true; uint32_t stage_mask = 7;  // debug: 1 front stages, 2 k_pack_tma, 4 k_pack_slow
    // stream table (b2_stream_*): the device side in `sp`; the host keeps the keys (it picks the table slots) and the free pool slots
    StreamPass sp = {}; bool has_streams = false, stream_armed = false, stream_ran = false, stream_valid = false;
    uint32_t st_max = 0, st_open = 0; std::vector<long long> st_keys; std::vector<uint8_t> st_state; std::vector<uint32_t> st_pool, st_pool_free;
    void* d_st_block[10] = {}; void* h_st_mapped[5] = {}; uint32_t* h_st_cnts = nullptr; uint8_t* h_st_out = nullptr; uint8_t* h_st_ctl = nullptr; uint8_t* d_st_ctl = nullptr;
    b2_stream_msg* h_st_msgs = nullptr; b2_stream_event* h_st_events = nullptr; uint8_t* h_st_ctrl = nullptr; uint32_t* h_st_run_ctrl = nullptr;
    cudaEvent_t st_ev[6] = {};
    const uint8_t* st_input = nullptr;      // the input bytes of the last batch with a stream pass (B2_STREAM_W_FROM_MSG of IN_INPUT messages); null once overwritten
    // the sending side (b2_stream_write): staging of its own, grown on demand: [0] host-sourced payloads [1] frames [2] per-write
    // records and scratch [3] per-table-slot scratch; pinned: the records as the host resolved them, the counters
    void* d_sw[4] = {}; size_t sw_have[4] = {}; SwRec* h_sw_recs = nullptr; size_t h_sw_have = 0; uint32_t* h_sw_cnts = nullptr;
    cudaEvent_t sw_ev[8] = {}; bool sw_ran = false;
    // pinned host mirrors
    b2_run_status* h_run_status = nullptr; b2_msg_desc* h_msgs = nullptr; uint8_t* h_resp = nullptr;
    uint32_t* h_totals = nullptr; uint32_t* h_run_tile_base = nullptr;
    // current batch
    uint32_t n_runs = 0, n_tiles = 0, nbytes = 0, max_run_tiles = 0; uint64_t covered = 0;
    bool uploaded = false, executed = false;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[kMaxStages + 1];
    const char* stage_names[kMaxStages];
    int n_stages = 0;
    float last_kernel_ms = 0.f; uint32_t last_launches = 0;
    cudaEvent_t ev_first = nullptr, ev_last = nullptr; bool first_pending = true;
    bool profile_stages = false; bool allow_small = true; bool use_fused = true; bool fused_last = false; bool slow_heavy = false;   // slow_heavy: the previous batch sent > 1/8 of its messages to k_pack_slow (CRC'd / compressed traffic): the classic pipeline serves that better
    bool adaptive_tile = false; bool dense = false; uint32_t avg_frame = 0;   // tile size follows the message size of the previous batch      // per-stage events only when a harness asks for stage times
    // walk groups (k_tile_search / k_tile_walk, DESIGN §3): b2_set_walk_group's mode (0 auto, 1 off, 2..8 forced), the uploaded batch's
    // group size and group count (the heads follow tile_info in the meta block), and the group size the last launch used
    uint32_t walk_group_mode = 0, walk_group = 1, n_groups = 0, walk_group_last = 1; size_t meta_group_off = 0;
    // small-batch (latency) mode: one compact H2D block, one compact output block, one D2H, one sync
    uint8_t* d_meta = nullptr; uint8_t* h_meta = nullptr;       // [runs | run_tile_base]
    uint8_t* d_small = nullptr; uint8_t* h_small = nullptr;     // [totals | run_status | msgs | resp]
    bool small = false, small_copy_queued = false, use_fused_small = true; SmallLayout sm = {};
    // b2_resident_plan: the kernels of a fused pass as compiled (read at creation), and the SM they share
    b2_resident_kernel plan[kPlanKernels] = {}; uint32_t sm_regs = 0, sm_smem = 0, sm_warps = 0, sm_blocks = 0, block_smem_reserve = 0;
};

// What a call overwrites on the device, and so which saved state it forgets; every call that writes the context's buffers says so first.
// kDevInput, the input (d_bytes, d_meta): the last h2 batch b2_h2_pack_responses reads zero-copy, and the input copy B2_STREAM_W_FROM_MSG
// reads (a B2_INPUT_PULL batch was read in the caller's region, which stays).  kDevBatch, the results and scratch: the uploaded batch.
enum : unsigned { kDevInput = 1, kDevBatch = 2 };
static void overwrites(b2_ctx* c, unsigned what) {
    if (what & kDevInput) { c->h2_last_in = 0; c->h2_last_out = 0; if (c->st_input == c->d_bytes) c->st_input = nullptr; }
    if (what & kDevBatch) { c->uploaded = false; c->executed = false; }
}

static uint32_t g_crc_tab_host[256];
static void crc_table_init() {
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0x82f63b78u : (c >> 1);
        g_crc_tab_host[i] = c;
    }
}

extern "C" const char* b2_last_error(void) { return g_err; }
extern "C" const char* b2_version(void) { return "brpc_b200 0.1 (sm_90a)"; }

// ---- pinned block pool (seam 3: butil::iobuf::blockmem_allocate / blockmem_deallocate, src/butil/iobuf.cpp:168-169; same role as
// rdma::block_pool, src/brpc/rdma/block_pool.h:74-105).  cudaHostAlloc / cudaFreeHost cost tens of microseconds and serialise
// with the device, so they are paid per SLAB, never per block: blocks of up to 8 KiB (IOBuf::DEFAULT_BLOCK_SIZE) are carved out
// of 4 MiB slabs and recycled through a free list; larger requests (socket read arenas, batch buffers) are rounded up to a power
// of two (+ 1 KiB of slack so 16-byte over-reads of a device kernel stay inside the mapping) and cached per size class when
// freed.  All memory is mapped (cudaHostAllocMapped | Portable): a kernel can read it in place (B2_INPUT_PULL).
namespace {
struct BlockPool {
    std::mutex mu;
    static constexpr size_t kSmall = 8192, kSlab = 4u << 20;
    std::vector<uint8_t*> slabs; std::vector<void*> small_free;
    std::unordered_map<void*, int> large_class;          // live + cached large blocks -> size class (log2)
    std::vector<void*> large_free[40];
    uint64_t n_host_alloc = 0;
    void* alloc(size_t size) {
        std::lock_guard<std::mutex> g(mu);
        if (size <= kSmall) {
            if (small_free.empty()) {
                uint8_t* slab = nullptr;
                if (cudaHostAlloc((void**)&slab, kSlab, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return nullptr;
                n_host_alloc++; slabs.push_back(slab);
                for (size_t o = 0; o + kSmall <= kSlab; o += kSmall) small_free.push_back(slab + o);
            }
            void* p = small_free.back(); small_free.pop_back(); return p;
        }
        int cls = 14; while (((size_t)1 << cls) < size) cls++;
        if (cls >= 40) return nullptr;
        if (!large_free[cls].empty()) { void* p = large_free[cls].back(); large_free[cls].pop_back(); return p; }
        void* p = nullptr;
        if (cudaHostAlloc(&p, ((size_t)1 << cls) + 1024, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return nullptr;
        n_host_alloc++; large_class[p] = cls;
        return p;
    }
    void free(void* p) {
        std::lock_guard<std::mutex> g(mu);
        auto it = large_class.find(p);
        if (it != large_class.end()) { large_free[it->second].push_back(p); return; }
        small_free.push_back(p);                           // (a slab block; slabs live until process exit)
    }
};
BlockPool& block_pool() { static BlockPool* p = new BlockPool; return *p; }
}
extern "C" void* b2_block_alloc(size_t size) {
    void* p = block_pool().alloc(size ? size : 1);
    if (!p) set_err("cudaHostAlloc failed");
    return p;
}
extern "C" void b2_block_free(void* p) { if (p) block_pool().free(p); }
extern "C" uint64_t b2_block_pool_host_allocs(void) { std::lock_guard<std::mutex> g(block_pool().mu); return block_pool().n_host_alloc; }

static void ring_halt(b2_ctx* c);
static void stream_free(b2_ctx* c);
static bool ring_busy(const b2_ctx* c) { for (uint32_t k = 0; k < kRingSlots; k++) if (!c->ring_collected[k]) return true; return false; }
static uint8_t* ring_slot(const b2_ctx* c, uint32_t ticket) { return c->ring_slots + (size_t)(ticket % kRingSlots) * c->ring_stride; }
// Every call that uploads to the context or touches h2 state is refused while a ticket of an h2 ring (k_h2_ring or k_h2_client_ring), of
// the client ring (k_ring<RingBody::requests>) or of the turn ring (k_ring<RingBody::replies>) is outstanding: the ticket uses the same
// device scratch and connection state.  A call that writes h2
// connection state also retires an h2 ring's resident kernel first: that CTA reads the state through L1, and a launch boundary is where
// L1 is known not to hold lines another kernel wrote since.
static bool ring_refuses(b2_ctx* c, bool writes_h2_state) {
    const RingKind k = c->ring_kind;
    if (k != RingKind::h2_server && k != RingKind::h2_client && !ring_packs(k)) return false;
    if (ring_busy(c)) {
        set_err(k == RingKind::h2_server ? "an h2 ring ticket is outstanding: b2_h2_ring_wait it first" :
                k == RingKind::h2_client ? "an h2 client ring ticket is outstanding: b2_h2_client_ring_wait it first" :
                k == RingKind::batch_client ? "a client ring ticket is outstanding: b2_client_ring_wait it first" :
                                              "a ring turn is outstanding: b2_ring_turn_wait it first");
        return true;
    }
    if (writes_h2_state && !ring_packs(k)) ring_halt(c);
    return false;
}
extern "C" void b2_ctx_destroy(b2_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->opt.device);
    ring_halt(c);
    if (c->ring_stream) cudaStreamDestroy(c->ring_stream);
    if (c->ring_slots) cudaFreeHost(c->ring_slots);
    if (c->ring_ctl) cudaFreeHost((void*)c->ring_ctl);
    cudaFree(c->d_ring_ticket); cudaFree(c->h2t_dev.turn);
    cudaFree(c->d_bytes); cudaFree(c->d_runs); cudaFree(c->d_run_tile_base); cudaFree(c->d_tiles); cudaFree(c->d_tile_base); cudaFree(c->d_tile_scratch); cudaFree(c->d_head_recs); cudaFree(c->d_tile_spec);
    cudaFree(c->d_run_status); cudaFree(c->d_frame_off); cudaFree(c->d_frame_run); cudaFree(c->d_msgs); cudaFree(c->d_aux); cudaFree(c->d_jobs); cudaFree(c->d_slow_idx); cudaFree(c->d_heads); cudaFree(c->d_slot);
    cudaFree(c->d_scan_tmp); cudaFree(c->d_resp); cudaFree(c->d_unz); cudaFree(c->d_snappy_tab); cudaFree(c->d_refs); cudaFree(c->d_iov); cudaFreeHost(c->h_iov); cudaFree(c->d_frame_row); cudaFree(c->d_rows); cudaFreeHost(c->h_refs); cudaFree(c->d_hpack); cudaFree(c->d_h2); cudaFree(c->d_h2_streams); cudaFree(c->d_h2_slots); cudaFree(c->d_h2_gz_merge); cudaFree(c->d_counters); cudaFree(c->d_totals); cudaFree(c->d_methods); cudaFree(c->d_crc_adv); cudaFree(c->d_meta); cudaFree(c->d_small); cudaFreeHost(c->h_meta); cudaFreeHost(c->h_small);
    cudaFreeHost(c->h_run_status); cudaFreeHost(c->h_msgs); cudaFreeHost(c->h_resp); cudaFreeHost(c->h_totals);
    cudaFreeHost(c->h_run_tile_base);
    stream_free(c);
    for (int i = 0; i <= kMaxStages; i++) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" int b2_ctx_create(const b2_options* o, b2_ctx** out) {
    if (!o || !out) { set_err("null argument"); return B2_E_INVAL; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_err("no CUDA device: brpc_b200 has no CPU path"); return B2_E_NO_DEVICE;
    }
    if (o->device < 0 || o->device >= ndev) { set_err("bad device ordinal"); return B2_E_INVAL; }
    if (o->max_batch_bytes == 0 || o->max_batch_bytes >= (1u << 31) || o->max_msgs == 0 || o->max_runs == 0) {
        set_err("capacities must be non-zero and max_batch_bytes < 2 GiB"); return B2_E_INVAL;
    }
    CU(cudaSetDevice(o->device));
    b2_ctx* c = new b2_ctx();
    { int v = 132; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, o->device); c->n_sms = (uint32_t)v; }
    for (int i = 0; i <= kMaxStages; i++) c->ev[i] = nullptr;
    c->opt = *o;
    c->adaptive_tile = o->tile_bytes == 0;
    uint32_t tile = o->tile_bytes ? o->tile_bytes : 8192;
    if (tile < 512 || (tile & (tile - 1))) { delete c; set_err("tile_bytes must be a power of two >= 512"); return B2_E_INVAL; }
    c->opt.tile_bytes = tile;
    if (c->opt.max_resp_bytes == 0) {
        uint64_t r = (uint64_t)o->max_batch_bytes + (uint64_t)o->max_msgs * 64 + (1u << 20);
        c->opt.max_resp_bytes = r > 0xfffffff0ull ? 0xfffffff0u : (uint32_t)r;
    }
    memset(&c->cfg, 0, sizeof c->cfg);
    c->cfg.max_body_size = o->max_body_size ? o->max_body_size : (64ull << 20);
    c->cfg.proto_mask = kProtoMaskDefault;
    c->cfg.tile_bytes = tile;
    c->cfg.tile_shift = 0; while ((1u << c->cfg.tile_shift) < tile) c->cfg.tile_shift++;
    c->max_tiles = o->max_batch_bytes / tile + o->max_runs + 1;
    const uint32_t scan_blocks = o->max_msgs / (kScanBlock * kScanItems) + 2;
#define ALLOC(ptr, bytes) do { if (cudaMalloc((void**)&(ptr), (bytes)) != cudaSuccess) { set_err("cudaMalloc %s failed", #ptr); b2_ctx_destroy(c); return B2_E_NOMEM; } } while (0)
#define HALLOC(ptr, bytes) do { if (cudaHostAlloc((void**)&(ptr), (bytes), cudaHostAllocDefault) != cudaSuccess) { set_err("cudaHostAlloc %s failed", #ptr); b2_ctx_destroy(c); return B2_E_NOMEM; } } while (0)
    ALLOC(c->d_bytes, (size_t)o->max_batch_bytes + 1024);
    ALLOC(c->d_runs, sizeof(b2_run) * (size_t)o->max_runs);
    ALLOC(c->d_run_tile_base, 4 * ((size_t)o->max_runs + 1));
    ALLOC(c->d_tiles, sizeof(TileRec) * (size_t)c->max_tiles);
    ALLOC(c->d_tile_base, 4 * (size_t)c->max_tiles);
    ALLOC(c->d_tile_scratch, 12 * (size_t)c->max_tiles);
    ALLOC(c->d_head_recs, sizeof(TileRec) * (size_t)c->max_tiles);
    {   // kSpecK offsets per tile; dense mode (tiles >= 2 KiB holding many small frames) keeps kSpecKDense
        size_t dense_tiles = (size_t)o->max_batch_bytes / 2048 + o->max_runs + 1; if (dense_tiles > c->max_tiles) dense_tiles = c->max_tiles;
        size_t words = (size_t)kSpecK * c->max_tiles; if ((size_t)kSpecKDense * dense_tiles > words) words = (size_t)kSpecKDense * dense_tiles;
        ALLOC(c->d_tile_spec, 4 * words);
    }
    ALLOC(c->d_run_status, sizeof(b2_run_status) * (size_t)o->max_runs);
    ALLOC(c->d_frame_off, 4 * (size_t)o->max_msgs);
    ALLOC(c->d_frame_run, 4 * (size_t)o->max_msgs);
    ALLOC(c->d_msgs, sizeof(b2_msg_desc) * (size_t)o->max_msgs);
    ALLOC(c->d_aux, sizeof(MsgAux) * (size_t)o->max_msgs);
    ALLOC(c->d_jobs, sizeof(PackJob) * (size_t)o->max_msgs);
    ALLOC(c->d_refs, sizeof(uint4) * (size_t)o->max_msgs);
    ALLOC(c->d_slow_idx, sizeof(uint32_t) * (size_t)o->max_msgs);
    ALLOC(c->d_heads, (size_t)kHeadBytes * (size_t)o->max_msgs);
    ALLOC(c->d_slot, 4 * ((size_t)o->max_msgs + 1));
    ALLOC(c->d_scan_tmp, 4 * (size_t)scan_blocks);
    ALLOC(c->d_resp, (size_t)c->opt.max_resp_bytes + 1024);
    ALLOC(c->d_unz, 2 * (size_t)c->opt.max_resp_bytes + 1024);
    ALLOC(c->d_snappy_tab, (size_t)kSnappyWarps * kSnappyMaxTable * 2);
    ALLOC(c->d_hpack, sizeof(HpackState) * (size_t)B2_HPACK_MAX_CONNS);
    CU(cudaMemset(c->d_hpack, 0, sizeof(HpackState) * (size_t)B2_HPACK_MAX_CONNS));
    ALLOC(c->d_counters, 8 * B2_N_COUNTERS);
    ALLOC(c->d_totals, 64);
    ALLOC(c->d_methods, sizeof(DevMethod) * 64);
    ALLOC(c->d_crc_adv, (kCrcHotWords + kCrcTreeWords) * 4);
    ALLOC(c->d_meta, (size_t)o->max_runs * 28 + 36 * (size_t)c->max_tiles + 64);
    ALLOC(c->d_small, kSmallBlock);
    HALLOC(c->h_meta, (size_t)o->max_runs * 28 + 36 * (size_t)c->max_tiles + 64);
    HALLOC(c->h_small, kSmallBlock);
    HALLOC(c->h_run_status, sizeof(b2_run_status) * (size_t)o->max_runs);
    HALLOC(c->h_msgs, sizeof(b2_msg_desc) * (size_t)o->max_msgs);
    HALLOC(c->h_refs, sizeof(b2_resp_ref) * (size_t)o->max_msgs);
    HALLOC(c->h_resp, (size_t)c->opt.max_resp_bytes);
    HALLOC(c->h_totals, 64);
    HALLOC(c->h_run_tile_base, 4 * ((size_t)o->max_runs + 1));
    CU(cudaMemset(c->d_counters, 0, 8 * B2_N_COUNTERS));
    CU(cudaMemset(c->d_bytes, 0, (size_t)o->max_batch_bytes + 1024));
    CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    for (int i = 0; i <= kMaxStages; i++) CU(cudaEventCreate(&c->ev[i]));
    CU(cudaEventCreate(&c->ev_first)); CU(cudaEventCreate(&c->ev_last));
    crc_table_init();
    CU(cudaMemcpyToSymbol(c_crc_table, g_crc_tab_host, sizeof g_crc_tab_host));
    {   // warp-CRC tables: T[k][b] = byte b followed by k zero bytes (k = 0..15), A512 = advance by 512 zero bytes,
        // tree t = advance by 16 << t zero bytes; the advance operators are stored byte-sliced (4 x 256)
        std::vector<uint32_t> tab(kCrcHotWords + kCrcTreeWords);
        auto adv = [&](uint32_t x, int bytes) { for (int k = 0; k < bytes; k++) x = g_crc_tab_host[x & 0xff] ^ (x >> 8); return x; };
        for (int k = 0; k < 16; k++) for (uint32_t b = 0; b < 256; b++) tab[k * 256 + b] = adv(g_crc_tab_host[b], k);
        for (int j = 0; j < 4; j++) for (uint32_t b = 0; b < 256; b++) tab[(16 + j) * 256 + b] = adv(b << (8 * j), 512);
        for (int t = 0; t < 5; t++) for (int j = 0; j < 4; j++) for (uint32_t b = 0; b < 256; b++)
            tab[kCrcHotWords + (t * 4 + j) * 256 + b] = adv(b << (8 * j), 16 << t);
        CU(cudaMemcpy(c->d_crc_adv, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
    }
    CU(cudaFuncSetAttribute(k_resolve, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CU(cudaFuncSetAttribute(k_pack_slow<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(8 * kSnapRing)));
    CU(cudaFuncSetAttribute(k_pack_tma<kPackGroup>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(PackWarpSmem) * kPackWarps)));
    CU(cudaFuncSetAttribute(k_pack_tma<kPackGroupSmall>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(PackWarpSmem) * kPackWarps)));
    if (const char* e = getenv("B2_PACK")) c->use_tma_pack = strcmp(e, "reg") != 0;
    if (const char* e = getenv("B2_SMALL")) c->use_fused_small = strcmp(e, "off") != 0;
    if (const char* e = getenv("B2_FUSED")) c->use_fused = strcmp(e, "off") != 0;
    CU(cudaFuncSetAttribute(k_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(FusedWarpSmem) * (kFusedWarps > kFusedWarpsDense ? kFusedWarps : kFusedWarpsDense))));
    CU(cudaFuncSetAttribute(k_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallSmem)));
#if defined(__NVCC__)       // (the host build of this file on the CUDA emulator, tests/cpp, has no function attributes: its plan stays empty)
    {
        const void* fn[kPlanKernels] = { (const void*)k_fused, (const void*)k_tile_search, (const void*)k_tile_walk, (const void*)k_resolve, (const void*)k_pack_slow<true> };
        const char* name[kPlanKernels] = { "k_fused", "k_tile_search", "k_tile_walk", "k_resolve", "k_pack_slow<true>" };
        const uint32_t threads[kPlanKernels] = { 0, kSearchThreadsFused, 128, 256, kSlowLiteThreads };     // (k_fused: by the batch's shape)
        for (int k = 0; k < kPlanKernels; k++) {
            cudaFuncAttributes a;
            CU(cudaFuncGetAttributes(&a, fn[k]));
            c->plan[k].name = name[k]; c->plan[k].regs = (uint32_t)a.numRegs; c->plan[k].threads = threads[k]; c->plan[k].smem_bytes = (uint32_t)a.sharedSizeBytes;
        }
        int v[5] = {};
        CU(cudaDeviceGetAttribute(&v[0], cudaDevAttrMaxRegistersPerMultiprocessor, o->device));
        CU(cudaDeviceGetAttribute(&v[1], cudaDevAttrMaxSharedMemoryPerMultiprocessor, o->device));
        CU(cudaDeviceGetAttribute(&v[2], cudaDevAttrMaxThreadsPerMultiProcessor, o->device));
        CU(cudaDeviceGetAttribute(&v[3], cudaDevAttrMaxBlocksPerMultiprocessor, o->device));
        CU(cudaDeviceGetAttribute(&v[4], cudaDevAttrReservedSharedMemoryPerBlock, o->device));
        c->sm_regs = (uint32_t)v[0]; c->sm_smem = (uint32_t)v[1]; c->sm_warps = (uint32_t)v[2] / 32; c->sm_blocks = (uint32_t)v[3]; c->block_smem_reserve = (uint32_t)v[4];
    }
#endif
    *out = c;
    return B2_OK;
}

extern "C" int b2_set_server_identity(b2_ctx* c, const char* ip_port) {
    if (!c) return B2_E_INVAL;
    if (ring_refuses(c, true)) return B2_E_INVAL;              // (the identity is a launch argument of k_h2_ring)
    const size_t n = ip_port ? strlen(ip_port) : 0;
    if (n >= sizeof c->cfg.identity) { set_err("identity too long"); return B2_E_INVAL; }
    memset(c->cfg.identity, 0, sizeof c->cfg.identity);
    if (n) memcpy(c->cfg.identity, ip_port, n);
    c->cfg.identity_len = (uint32_t)n;
    return B2_OK;
}

extern "C" int b2_set_modes(b2_ctx* c, int input_mode, int resp_mode) {
    if (!c || (input_mode != B2_INPUT_COPY && input_mode != B2_INPUT_PULL) || (resp_mode != B2_RESP_COPY && resp_mode != B2_RESP_BY_REF && resp_mode != B2_RESP_IOVEC)) { set_err("bad mode"); return B2_E_INVAL; }
    static_assert(sizeof(b2_resp_ref) == sizeof(uint4), "b2_resp_ref is 16 bytes");
    static_assert(sizeof(b2_iovec) == sizeof(ulonglong2) && sizeof(void*) == 8, "b2_iovec is a 16-byte struct iovec");
    if (resp_mode == B2_RESP_IOVEC && !c->d_iov) {
        CU(cudaSetDevice(c->opt.device));
        if (cudaMalloc((void**)&c->d_iov, 32 * (size_t)c->opt.max_msgs) != cudaSuccess || cudaHostAlloc((void**)&c->h_iov, 32 * (size_t)c->opt.max_msgs, cudaHostAllocDefault) != cudaSuccess) {
            cudaFree(c->d_iov); c->d_iov = nullptr; cudaGetLastError(); set_err("allocation of the iovec list failed"); return B2_E_NOMEM;
        }
    }
    if (input_mode == B2_INPUT_PULL && !c->d_rows) {
        // row stash of the pull walk: spec_k rows of 128 bytes per tile (tiles are >= 32 KiB in this mode unless the caller fixed them)
        CU(cudaSetDevice(c->opt.device));
        const uint32_t tile = c->adaptive_tile ? 32768u : c->opt.tile_bytes;
        const size_t tiles = (size_t)c->opt.max_batch_bytes / tile + c->opt.max_runs + 1;
        const size_t rows = tiles * (tile >= 2048 ? kSpecKDense : kSpecK);
        if (cudaMalloc((void**)&c->d_rows, rows * 128) != cudaSuccess || cudaMalloc((void**)&c->d_frame_row, 4 * (size_t)c->opt.max_msgs) != cudaSuccess) {
            cudaFree(c->d_rows); c->d_rows = nullptr; cudaGetLastError(); set_err("cudaMalloc of the pull-mode row stash failed"); return B2_E_NOMEM;
        }
    }
    ring_halt(c);
    c->input_mode = input_mode; c->resp_mode = resp_mode; c->cfg.by_ref = resp_mode != B2_RESP_COPY; c->cfg.pull = input_mode == B2_INPUT_PULL; c->cfg.pull_vecs = resp_mode != B2_RESP_COPY ? 6u : 8u;
    overwrites(c, kDevBatch);                       // (the uploaded batch was laid out for the old modes)
    return B2_OK;
}

extern "C" int b2_set_protocols(b2_ctx* c, uint32_t mask) {
    const uint32_t known = (1u << 1) | (1u << 2) | (1u << 3) | (1u << 4) | (1u << 12);
    if (!c || mask == 0 || (mask & ~known)) { set_err("unknown protocol in mask (baidu_std 1, streaming_rpc 2, hulu_pbrpc 3, sofa_pbrpc 4, nshead 12)"); return B2_E_INVAL; }
    ring_halt(c);
    c->cfg.proto_mask = mask;
    return B2_OK;
}

extern "C" int b2_set_stream_handler(b2_ctx* c, int kind) {
    if (!c || (kind != B2_STREAM_DESC_ONLY && kind != B2_STREAM_SNAPPY_UNCOMPRESS)) { set_err("bad stream handler"); return B2_E_INVAL; }
    c->cfg.stream_handler = (uint32_t)kind;
    return B2_OK;
}

extern "C" int b2_register_method(b2_ctx* c, const b2_method* m) {
    if (!c || !m || !m->service_full_name || !m->service_name || !m->method_name || !m->request_type_name) { set_err("null argument"); return B2_E_INVAL; }
    if (c->methods.size() >= 64) { set_err("method table full"); return B2_E_CAPACITY; }
    DevMethod d; memset(&d, 0, sizeof d);
    std::string full = std::string(m->service_full_name) + "." + m->method_name;
    if (full.size() >= sizeof d.full_method || strlen(m->service_name) >= sizeof d.service_short ||
        strlen(m->service_full_name) >= sizeof d.service_full || strlen(m->request_type_name) >= sizeof d.request_type) {
        set_err("method names too long"); return B2_E_INVAL;
    }
    memcpy(d.full_method, full.data(), full.size()); d.full_method_len = (uint32_t)full.size();
    d.service_short_len = (uint32_t)strlen(m->service_name); memcpy(d.service_short, m->service_name, d.service_short_len);
    d.service_full_len = (uint32_t)strlen(m->service_full_name); memcpy(d.service_full, m->service_full_name, d.service_full_len);
    d.request_type_len = (uint32_t)strlen(m->request_type_name); memcpy(d.request_type, m->request_type_name, d.request_type_len);
    d.handler = m->handler; d.echo_attachment = m->echo_attachment;
    d.response_checksum_type = m->response_checksum_type; d.response_compress_type = m->response_compress_type;
    ring_halt(c);                                  // (DevConfig is a launch argument of the resident kernel)
    c->methods.push_back(d);
    c->cfg.n_methods = (uint32_t)c->methods.size();
    CU(cudaSetDevice(c->opt.device));
    CU(cudaMemcpy(c->d_methods, c->methods.data(), sizeof(DevMethod) * c->methods.size(), cudaMemcpyHostToDevice));
    return (int)c->methods.size() - 1;
}

static BatchPtrs make_ptrs(b2_ctx* c) {
    BatchPtrs B;
    B.bytes = c->d_bytes; B.runs = c->d_runs; B.run_tile_base = c->d_run_tile_base; B.tiles = c->d_tiles;
    B.tile_base = c->d_tile_base; B.tile_scratch = c->d_tile_scratch; B.tile_spec = c->d_tile_spec; B.run_status = c->d_run_status; B.frame_off = c->d_frame_off; B.frame_run = c->d_frame_run; B.frame_row = c->d_frame_row; B.rows = c->d_rows; B.msgs = c->d_msgs;
    B.aux = c->d_aux; B.jobs = c->d_jobs; B.refs = c->d_refs; B.slow_idx = c->d_slow_idx; B.heads = c->d_heads; B.slot = c->d_slot; B.scan_tmp = c->d_scan_tmp; B.resp = c->d_resp; B.unz = c->d_unz; B.snappy_tab = c->d_snappy_tab; B.counters = c->d_counters;
    B.totals = c->d_totals; B.methods = c->d_methods; B.crc_adv = c->d_crc_adv;
    B.n_runs = c->n_runs; B.n_tiles = c->n_tiles; B.max_msgs = c->opt.max_msgs; B.max_resp = c->opt.max_resp_bytes;
    B.runs = reinterpret_cast<const b2_run*>(c->d_meta);
    B.run_tile_base = reinterpret_cast<const uint32_t*>(c->d_meta + (size_t)c->n_runs * sizeof(b2_run));
    B.tile_info = reinterpret_cast<const uint4*>(c->d_meta + c->meta_tile_off);
    B.group_heads = reinterpret_cast<const uint32_t*>(c->d_meta + c->meta_group_off + 16 * (size_t)c->n_groups); B.head_recs = c->d_head_recs;
    B.n_groups = c->n_groups; B.walk_group = 1;     // (launch_pipeline groups)
    if (c->input_mode == B2_INPUT_PULL) B.bytes = c->pull_bytes;          // the caller's pinned + mapped batch buffer, read in place
    if (c->small) {
        B.refs = reinterpret_cast<uint4*>(c->d_small + c->sm.off_refs);
        B.totals = reinterpret_cast<uint32_t*>(c->d_small);
        B.run_status = reinterpret_cast<b2_run_status*>(c->d_small + c->sm.off_rs);
        B.msgs = reinterpret_cast<b2_msg_desc*>(c->d_small + c->sm.off_msgs);
        B.resp = c->d_small + c->sm.off_resp;
        B.max_msgs = c->sm.msgs; B.max_resp = c->sm.resp;
    }
    return B;
}

// The fused decode+pack kernel serves batches whose bytes and replies both live in HBM
static bool takes_fused(const b2_ctx* c) {
    return c->use_fused && !c->slow_heavy && !c->small && c->input_mode == B2_INPUT_COPY && c->resp_mode == B2_RESP_COPY && c->use_tma_pack &&
           (((uint64_t)c->nbytes + 255) & ~255ull) + 4096 <= c->opt.max_resp_bytes;
}
// Walk group of an uploaded batch.  Auto: 2 tiles on the fused path once the frame size is known and frames are not dense — the search
// then reads half the windows, and the walk's longer chain still ends under the other batch's k_fused (4 and 8 tiles were slower on the
// bench batch, DESIGN §9.1) — else 1 (pull mode keeps its own walk).
static uint32_t pick_walk_group(const b2_ctx* c) {
    if (c->input_mode == B2_INPUT_PULL || c->walk_group_mode == 1) return 1;
    if (c->walk_group_mode >= 2) return c->walk_group_mode;
    return takes_fused(c) && c->avg_frame && !c->dense ? 2u : 1u;
}

extern "C" int b2_batch_upload(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs) {
    if (!c || (!bytes && nbytes) || (!runs && n_runs)) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    // (B2_INPUT_PULL: `bytes` is the caller's whole pinned arena and nothing is copied — what is bounded is the bytes the runs cover)
    if ((c->input_mode != B2_INPUT_PULL && nbytes > c->opt.max_batch_bytes) || nbytes >= (1u << 31) || n_runs > c->opt.max_runs) { set_err("batch exceeds ctx capacity"); return B2_E_CAPACITY; }
    uint64_t covered = 0; for (uint32_t r = 0; r < n_runs; r++) covered += runs[r].length;
    if (c->input_mode == B2_INPUT_PULL && covered > c->opt.max_batch_bytes) { set_err("runs exceed ctx capacity"); return B2_E_CAPACITY; }
    c->stream_valid = false; c->st_view_ticket = 0;
    c->covered = covered;                           // (what the runs hold: with B2_INPUT_PULL nbytes spans the caller's whole arena)
    CU(cudaSetDevice(c->opt.device));
    if (!c->avg_frame && n_runs && runs[0].length >= 12 && (uint64_t)runs[0].offset + 12 <= nbytes) {
        // a context that has not finished a batch yet takes the frame size from the first baidu_std / streaming_rpc header of the batch, so
        // that its tiles and k_fused's shape follow the traffic from the first batch on (a context whose passes are only launched and
        // waited for never downloads a batch; its k_fused would keep the dense shape, which leaves no room for the other batch's kernels)
        const uint8_t* f = static_cast<const uint8_t*>(bytes) + runs[0].offset;
        uint32_t w[2]; memcpy(w, f, 8);
        const uint32_t body = __builtin_bswap32(w[1]);
        if ((w[0] == kMagicPRPC || w[0] == kMagicSTRM) && body <= c->cfg.max_body_size && body < (1u << 30)) c->avg_frame = 12 + body;
    }
    if (c->adaptive_tile) {
        // like Socket::_avg_msg_size steering the read size (input_messenger.cpp:348-353): a tile should hold
        // 6-12 messages so the speculative entry search reads a small fraction of it
        uint32_t t = 8192;
        // (B2_INPUT_PULL: the speculative scan window of every tile crosses PCIe, so tiles are 4x larger)
        const uint32_t per_tile = c->input_mode == B2_INPUT_PULL ? 48u : 6u;
        if (c->input_mode == B2_INPUT_PULL && t < 32768) t = 32768;
        while (t < (1u << 20) && t < per_tile * c->avg_frame) t <<= 1;
        c->cfg.tile_bytes = t; c->cfg.tile_shift = 0; while ((1u << c->cfg.tile_shift) < t) c->cfg.tile_shift++;
    }
    const uint32_t shift = c->cfg.tile_shift, tile = c->cfg.tile_bytes;
    // small requests (the previous batches' average says a tile holds more than kSpecK frames): k_tile_walk keeps longer offset
    // lists so that k_frame_table still only copies (a measured 139 -> 29 us for 124-byte frames)
    c->dense = tile >= 2048 && c->avg_frame && (uint64_t)c->avg_frame * kSpecK < tile;
    c->cfg.spec_k = c->dense ? kSpecKDense : kSpecK;
    uint64_t nt = 0; uint32_t max_rt = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        if ((runs[r].offset & 15u) || (uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run offset must be 16-aligned and inside the batch"); return B2_E_INVAL; }
        c->h_run_tile_base[r] = (uint32_t)nt;
        const uint32_t t = (uint32_t)(((uint64_t)runs[r].length + tile - 1) >> shift);
        nt += t; if (t > max_rt) max_rt = t;
    }
    c->h_run_tile_base[n_runs] = (uint32_t)nt;
    if (nt > c->max_tiles) { set_err("too many tiles"); return B2_E_CAPACITY; }
    c->n_runs = n_runs; c->n_tiles = (uint32_t)nt; c->nbytes = nbytes; c->max_run_tiles = max_rt; c->host_bytes = bytes;
    // latency path: outputs of a small batch live in one compact block -> one D2H copy, one sync
    c->small = c->allow_small && nbytes <= kSmallBytes && n_runs <= kSmallRuns && n_runs > 0;
    c->walk_group = pick_walk_group(c);
    // runs + tile bases travel as one compact block (24 B * n is 4-byte aligned), then the tile records, and with walk groups the
    // heads' tile records (k_tile_search's tiles) and tile indices
    const size_t tile_off = ((size_t)n_runs * sizeof(b2_run) + 4 * ((size_t)n_runs + 1) + 15) & ~(size_t)15;
    c->meta_tile_off = tile_off; c->meta_group_off = tile_off + 16 * (size_t)nt;
    uint32_t ng = 0;
    if (c->walk_group > 1)
        for (uint32_t r = 0; r < n_runs; r++) ng += (c->h_run_tile_base[r + 1] - c->h_run_tile_base[r] + c->walk_group - 1) / c->walk_group;
    c->n_groups = ng;
    const size_t meta_bytes = c->meta_group_off + 20 * (size_t)ng;
    if (n_runs) memcpy(c->h_meta, runs, (size_t)n_runs * sizeof(b2_run));
    memcpy(c->h_meta + (size_t)n_runs * sizeof(b2_run), c->h_run_tile_base, 4 * ((size_t)n_runs + 1));
    {   // per-tile record {run offset, run length, tile index in the run, run | flags << 24}: one load per tile thread
        uint32_t* ti = reinterpret_cast<uint32_t*>(c->h_meta + tile_off);
        for (uint32_t r = 0; r < n_runs; r++) {
            const uint32_t t0 = c->h_run_tile_base[r], t1 = c->h_run_tile_base[r + 1];
            for (uint32_t t = t0; t < t1; t++) { uint32_t* q = ti + 4 * (size_t)t; q[0] = runs[r].offset; q[1] = runs[r].length; q[2] = t - t0; q[3] = r | (runs[r].flags << 24); }
        }
        uint32_t* hi = reinterpret_cast<uint32_t*>(c->h_meta + c->meta_group_off);
        uint32_t* heads = hi + 4 * (size_t)ng;
        uint32_t g = 0;
        if (c->walk_group > 1)
            for (uint32_t r = 0; r < n_runs; r++)
                for (uint32_t t = c->h_run_tile_base[r]; t < c->h_run_tile_base[r + 1]; t += c->walk_group, g++) { memcpy(hi + 4 * (size_t)g, ti + 4 * (size_t)t, 16); heads[g] = t; }
    }
    overwrites(c, kDevInput | kDevBatch);
    if (c->input_mode == B2_INPUT_PULL) {
        // no copy: the kernels read the caller's pinned block in place (it must stay untouched until collect)
        void* dp = nullptr;
        if (nbytes && cudaHostGetDevicePointer(&dp, const_cast<void*>(bytes), 0) != cudaSuccess) {
            cudaGetLastError(); set_err("B2_INPUT_PULL: bytes must be pinned + mapped memory from b2_block_alloc"); return B2_E_INVAL;
        }
        c->pull_bytes = static_cast<const uint8_t*>(dp);
    } else if (nbytes) CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_meta, c->h_meta, meta_bytes, cudaMemcpyHostToDevice, c->stream));
    if (c->small) c->sm = small_layout(nbytes, n_runs, c->opt.max_msgs);
    if (const char* e = getenv("B2_STAGE_MASK")) c->stage_mask = (uint32_t)atoi(e);   // timing experiments only (tools/overlap_probe.py)
    c->uploaded = true;
    return B2_OK;
}

// The stream pass of a batch call (k_stream_*): behind the stage that wrote msgs[], on the same stream, inside the call's synchronisation.
static const char* const kStreamStages[5] = { "stream_route", "stream_alloc", "stream_group", "stream_run", "stream_rst" };
static uint32_t grid(uint32_t items, uint32_t per_block, uint32_t most) { const uint32_t g = (items + per_block - 1) / per_block; return g < 1 ? 1u : g < most ? g : most; }
static int launch_stream_pass(b2_ctx* c, const BatchPtrs& B, cudaStream_t s, uint32_t& launches) {
    const StreamPass& S = c->sp;
    const uint32_t msg_bound = c->small ? c->sm.msgs : c->opt.max_msgs, sms = c->n_sms;
    CU(cudaMemsetAsync(S.cnts, 0, 4 * (16 + 2 * (size_t)S.cap), s));          // counters | cnt | fill
    CU(cudaEventRecord(c->st_ev[0], s));
    k_stream_route<<<grid(msg_bound, 256, sms * 4), 256, 0, s>>>(B, S); CU(cudaEventRecord(c->st_ev[1], s));
    k_stream_alloc<<<grid(c->st_max, 256, sms), 256, 0, s>>>(B, S); CU(cudaEventRecord(c->st_ev[2], s));
    k_stream_group<<<grid(msg_bound, 256, sms * 4), 256, 0, s>>>(B, S); CU(cudaEventRecord(c->st_ev[3], s));
    k_stream_run<<<grid(c->st_max, 4, sms * 8), 128, 0, s>>>(B, S); CU(cudaEventRecord(c->st_ev[4], s));
    k_stream_rst<<<grid(c->n_runs, 4, sms * 4), 128, 0, s>>>(B, S); CU(cudaEventRecord(c->st_ev[5], s));
    CU(cudaMemcpyAsync(c->h_st_cnts, S.cnts, 64, cudaMemcpyDeviceToHost, s));
    if (ring_runs_streams(c->ring_kind)) CU(cudaMemsetAsync(S.cnt, 0, 8 * (size_t)S.cap, s));     // cnt | fill: zero when the ring's next ticket starts
    launches += 5; c->stream_ran = true; c->st_input = B.bytes;
    return B2_OK;
}

// k_fused's warps per CTA for the uploaded batch (B2_FUSED_WARPS: the shape that leaves room for the other batch's kernels; the dense
// shape for small frames, or while the frame size is not known: a tile may then hold many frames to walk again)
static uint32_t fused_warps(const b2_ctx* c) { return c->avg_frame && !c->dense ? kFusedWarps : kFusedWarpsDense; }
// k_resolve's dynamic shared memory: every run's tile records, or none when some run does not fit (EVERY run of the launch then uses the
// global scratch).  Ahead of k_fused none either: the SM a k_fused CTA holds is configured for it (132 KB of shared memory for its 129),
// and a k_resolve block only starts beside it without records in shared memory.
static size_t resolve_smem(const b2_ctx* c, bool fused) { const size_t b = (size_t)c->max_run_tiles * 12; return fused || b > 200 * 1024 ? 0 : b; }

// timed: events around the pass (kernel_ms, b2_stage_times).  b2_batch_launch passes false: a record between two passes of a stream
// sits on the path from one pass's last kernel to the next pass's first, which runs beside the other stream's k_fused.
static int launch_pipeline(b2_ctx* c, bool timed = true) {
    BatchPtrs B = make_ptrs(c);
    DevConfig C = c->cfg;
    const bool fused = takes_fused(c);
    // the upload's walk groups, unless auto mode picked them for the fused path and this launch takes the slot-scan pipeline
    B.walk_group = fused || c->walk_group_mode >= 2 ? c->walk_group : 1u;
    c->walk_group_last = B.walk_group;
    C.fused = fused ? 1u : 0u; C.ovf_base = (c->nbytes + 255u) & ~255u; c->fused_last = fused;
    cudaStream_t s = c->stream;
    int st = 0; uint32_t launches = 0;
    const bool prof = c->profile_stages;
    auto mark = [&](const char* name) { if (prof) { c->stage_names[st] = name; cudaEventRecord(c->ev[st + 1], s); st++; } };
    const uint32_t mask = c->stage_mask;
    const bool small_launch = c->small && c->use_fused_small && !prof;
    // the pass's totals start at zero: k_tile_search zeroes them when it runs (a launch of the other batch's pass then no longer waits
    // for a memset and a second dependent launch behind it), a memset otherwise
    const bool search_zeroes = (mask & 1) && c->n_runs && c->n_tiles && !small_launch;
    if ((mask & 1) && !search_zeroes) CU(cudaMemsetAsync(B.totals, 0, 48, s));
    if (timed) CU(cudaEventRecord(c->ev[0], s));
    c->stream_ran = false;
    if (c->n_runs == 0) { c->n_stages = 0; c->last_launches = 0; return B2_OK; }
    if (small_launch) {
        // latency path: the whole pipeline in one launch, one CTA
        k_small<<<1, kSmallThreads, sizeof(SmallSmem), s>>>(B, C);
        launches = 1;
        if (c->stream_armed) { int rc = launch_stream_pass(c, B, s, launches); if (rc != B2_OK) return rc; }
        c->stage_names[0] = "fused_small";
        if (timed) cudaEventRecord(c->ev[1], s);
        c->n_stages = timed ? 1 : 0; c->last_launches = launches;
        CU(cudaGetLastError());
        return B2_OK;
    }
    const uint32_t sms = c->n_sms;
    if (mask & 1) {
    if (c->n_tiles) {
        // (ahead of k_fused, in blocks that start beside the other batch's k_fused: b2_resident_plan)
        const uint32_t search_threads = fused ? kSearchThreadsFused : 256u;
        BatchPtrs S = B;                            // (walk groups: only the heads are searched, their entries go to head_recs)
        if (B.walk_group > 1) { S.tile_info = reinterpret_cast<const uint4*>(c->d_meta + c->meta_group_off); S.tiles = B.head_recs; S.n_tiles = c->n_groups; }
        k_tile_search<<<(S.n_tiles * 32 + search_threads - 1) / search_threads, search_threads, 0, s>>>(S, C); launches++; mark("tile_search");
        if (C.pull) k_tile_walk_pull<<<(uint32_t)(((uint64_t)c->n_tiles * 8 + 127) / 128), 128, 0, s>>>(B, C);
        else if (B.walk_group > 1) k_tile_walk<<<(c->n_groups + kWalkGroupThreads - 1) / kWalkGroupThreads, kWalkGroupThreads, 0, s>>>(B, C);
        else k_tile_walk<<<(c->n_tiles + 127) / 128, 128, 0, s>>>(B, C);
        launches++; mark("tile_walk");
    }
    {
        const size_t smem = resolve_smem(c, fused);
        k_resolve<<<c->n_runs, 256, smem, s>>>(B, C, smem == 0 ? 1u : 0u); launches++; mark("resolve");
    }
    if (fused) {
        // one pass over the bytes: decode + echo + pack per live tile (k_frame_table / k_decode / k_scan / k_pack_tma are not needed)
        const uint32_t fw = fused_warps(c);
        if (c->n_tiles) { k_fused<<<sms, fw * 32, sizeof(FusedWarpSmem) * fw, s>>>(B, C); launches++; mark("fused"); }
    } else {
    if (c->n_tiles) { k_frame_table<<<(uint32_t)(((uint64_t)c->n_tiles * C.spec_k + 255) / 256), 256, 0, s>>>(B, C); launches++; mark("frame_table"); }
    // message-count dependent kernels are persistent: fixed grids (multiples of the SM count)
    // stride over the device-side message count, so no host round trip sizes a launch
    k_decode<<<sms * B2_DECODE_MIN_BLOCKS, kDecodeWarps * 32, 0, s>>>(B, C); launches++; mark("decode");
    k_scan_blocks<<<sms, kScanBlock, 0, s>>>(B); launches++;
    mark("scan");
    }
    }
    if (fused) {
        // (as many warps as k_pack_slow<false> gets, in blocks that start beside the other batch's k_fused)
        if (mask & 4) { k_pack_slow<true><<<sms * B2_SLOW_MIN_BLOCKS * (256 / kSlowLiteThreads), kSlowLiteThreads, 0, s>>>(B, C); launches++; mark("pack_slow"); }
    } else if (c->use_tma_pack) {
        // the verify pass decides which CRC-carrying echoes k_pack_tma may move; k_pack_slow answers the ones that fail
        if (mask & 4) {
            if (c->slow_heavy || c->cfg.by_ref) { C.verify_done = 1; k_crc_verify<<<sms * 6, 256, 0, s>>>(B, C); launches++; mark("crc_verify"); }
            k_pack_slow<false><<<sms * B2_SLOW_MIN_BLOCKS, 256, 8 * kSnapRing, s>>>(B, C); launches++; mark("pack_slow");
        }
        if (mask & 2) {
            // small requests: 32 messages per warp round instead of 8 (measured +30 % at 64 B payloads, -3 % at 1 KB)
            if ((c->avg_frame && c->avg_frame < 640) || c->cfg.by_ref) k_pack_tma<kPackGroupSmall><<<sms, kPackWarps * 32, sizeof(PackWarpSmem) * kPackWarps, s>>>(B, C);
            else k_pack_tma<kPackGroup><<<sms, kPackWarps * 32, sizeof(PackWarpSmem) * kPackWarps, s>>>(B, C);
            launches++; mark("pack");
        }
    } else { k_pack<<<sms * B2_PACK_MIN_BLOCKS, 256, 0, s>>>(B, C); launches++; mark("pack"); }
    if (c->resp_mode == B2_RESP_IOVEC && !c->small) {
        k_emit_iov<<<sms * 4, 256, 0, s>>>(B, c->d_iov, (unsigned long long)(uintptr_t)c->h_resp, (unsigned long long)(uintptr_t)c->host_bytes);
        launches++; mark("emit_iov");
    }
    if (c->stream_armed) { int rc = launch_stream_pass(c, B, s, launches); if (rc != B2_OK) return rc; }
    if (!prof && timed) { c->stage_names[0] = "pipeline"; cudaEventRecord(c->ev[1], s); st = 1; }
    c->n_stages = st; c->last_launches = launches;
    CU(cudaGetLastError());
    return B2_OK;
}

// b2_batch_execute / _execute_many / b2_batch_launch replay the uploaded batch, without its stream pass
static bool replay_refused(const b2_ctx* c) {
    if (!c || !c->uploaded) { set_err("no batch uploaded"); return true; }
    if (c->stream_armed) { set_err("a submitted batch of a context with a stream table must be collected first: this entry point replays a batch and does not run the stream pass"); return true; }
    return false;
}
extern "C" int b2_batch_execute(b2_ctx* c, float* kernel_ms, uint32_t* n_launches) {
    if (replay_refused(c)) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    c->profile_stages = true;
    int rc = launch_pipeline(c);
    c->profile_stages = false;
    if (rc != B2_OK) return rc;
    CU(cudaStreamSynchronize(c->stream));
    float ms = 0.f;
    if (c->n_stages) CU(cudaEventElapsedTime(&ms, c->ev[0], c->ev[c->n_stages]));
    c->last_kernel_ms = ms; c->executed = true;
    if (kernel_ms) *kernel_ms = ms;
    if (n_launches) *n_launches = c->last_launches;
    return B2_OK;
}

extern "C" int b2_batch_execute_many(b2_ctx* c, uint32_t steps, float* total_ms, uint32_t* n_launches) {
    if (steps == 0) { set_err("no batch uploaded"); return B2_E_INVAL; }
    if (replay_refused(c)) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    cudaEvent_t e0, e1;
    CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    CU(cudaEventRecord(e0, c->stream));
    uint32_t launches = 0;
    for (uint32_t i = 0; i < steps; i++) {
        int rc = launch_pipeline(c);
        if (rc != B2_OK) return rc;
        launches += c->last_launches;
    }
    CU(cudaEventRecord(e1, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    c->executed = true;
    if (c->n_stages) { float t = 0.f; cudaEventElapsedTime(&t, c->ev[0], c->ev[c->n_stages]); c->last_kernel_ms = t; }
    if (total_ms) *total_ms = ms;
    if (n_launches) *n_launches = launches;
    return B2_OK;
}

extern "C" int b2_batch_launch(b2_ctx* c) {
    if (replay_refused(c)) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    if (c->first_pending) { CU(cudaEventRecord(c->ev_first, c->stream)); c->first_pending = false; }
    int rc = launch_pipeline(c, false);
    if (rc != B2_OK) return rc;
    CU(cudaEventRecord(c->ev_last, c->stream));
    c->executed = true;
    return B2_OK;
}
extern "C" int b2_batch_wait(b2_ctx* c) {
    if (!c) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    CU(cudaStreamSynchronize(c->stream));
    c->first_pending = true;
    return B2_OK;
}
extern "C" int b2_elapsed_ms(b2_ctx* a, b2_ctx* b, float* ms) {
    if (!a || !b || !ms) return B2_E_INVAL;
    CU(cudaSetDevice(a->opt.device));
    CU(cudaEventElapsedTime(ms, a->ev_first, b->ev_last));
    return B2_OK;
}

// B2_RESP_IOVEC on the latency path (a handful of messages in one compact block): the list is built here from the refs that came back
static void refs_to_iov(b2_ctx* c, b2_batch_result* out, const void* host_bytes) {
    b2_run_status* rs = const_cast<b2_run_status*>(out->runs);
    for (uint32_t r = 0; r < out->n_runs; r++) rs[r].n_unanswered = 0;
    for (uint32_t i = 0; i < out->n_msgs; i++) {
        const b2_msg_desc& d = out->msgs[i];
        b2_iovec a = { const_cast<uint8_t*>(out->resp), 0 }, b = a;
        if (d.status == B2_MSG_ECHOED || d.status == B2_MSG_ERROR_REPLIED) {
            const b2_resp_ref rf = d.status == B2_MSG_ECHOED ? out->refs[i] : b2_resp_ref{0, 0, 0, 0};
            a.iov_base = const_cast<uint8_t*>(out->resp) + d.resp_off; a.iov_len = rf.src_len ? rf.prefix_len : d.resp_len;
            if (rf.src_len) { b.iov_base = const_cast<uint8_t*>(static_cast<const uint8_t*>(host_bytes)) + rf.src_off; b.iov_len = rf.src_len; }
        } else rs[d.run_idx].n_unanswered++;
        c->h_iov[2 * (size_t)i] = a; c->h_iov[2 * (size_t)i + 1] = b;
    }
    out->iov = c->h_iov; out->refs = nullptr;
}

static int download_normal(b2_ctx* c, b2_batch_result* out) {
    CU(cudaMemcpyAsync(c->h_totals, c->d_totals, 48, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (c->n_runs && c->fused_last) {
        // the fused kernel keeps slow replies in an overflow area behind the batch-shaped part of resp: traffic that is mostly
        // CRC'd / compressed / errors is better served (and may only fit) through the slot-scan pipeline
        const bool heavy = (uint64_t)c->h_totals[3] * 8 > c->h_totals[0];
        if ((c->h_totals[2] & 2u) && !(c->h_totals[2] & 1u)) {
            c->slow_heavy = true;
            int rc = launch_pipeline(c); if (rc != B2_OK) return rc;
            CU(cudaMemcpyAsync(c->h_totals, c->d_totals, 48, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
        }
        c->slow_heavy = heavy || c->slow_heavy;
    } else if (c->n_runs && c->slow_heavy && !c->small) {
        c->slow_heavy = ((uint64_t)c->h_totals[3] + c->h_totals[7]) * 8 > c->h_totals[0];   // ([7]: CRC-carrying echoes the classic pipeline verifies)
    }
    if (c->n_runs && (c->h_totals[2] & 3u)) {
        set_err(c->h_totals[2] & 1u ? "more messages than max_msgs" : "responses exceed max_resp_bytes"); return B2_E_CAPACITY;
    }
    // (k_fused / k_pack_slow: replies of parked messages are placed after the kernel's own end-of-area note, so the span is taken from the allocator)
    if (c->n_runs && c->fused_last) c->h_totals[1] = ((c->nbytes + 255u) & ~255u) + c->h_totals[9];
    const uint32_t n_msgs = c->n_runs ? c->h_totals[0] : 0, resp_bytes = c->n_runs ? c->h_totals[1] : 0;
    if (c->n_runs) CU(cudaMemcpyAsync(c->h_run_status, c->d_run_status, sizeof(b2_run_status) * c->n_runs, cudaMemcpyDeviceToHost, c->stream));
    if (n_msgs) CU(cudaMemcpyAsync(c->h_msgs, c->d_msgs, sizeof(b2_msg_desc) * (size_t)n_msgs, cudaMemcpyDeviceToHost, c->stream));
    if (resp_bytes) CU(cudaMemcpyAsync(c->h_resp, c->d_resp, resp_bytes, cudaMemcpyDeviceToHost, c->stream));
    const bool iovec = c->resp_mode == B2_RESP_IOVEC;
    if (n_msgs && c->cfg.by_ref && !iovec) CU(cudaMemcpyAsync(c->h_refs, c->d_refs, sizeof(b2_resp_ref) * (size_t)n_msgs, cudaMemcpyDeviceToHost, c->stream));
    if (n_msgs && iovec) CU(cudaMemcpyAsync(c->h_iov, c->d_iov, 32 * (size_t)n_msgs, cudaMemcpyDeviceToHost, c->stream));
    if (c->stream_ran && c->h_st_cnts[2]) CU(cudaMemcpyAsync(c->h_st_out, c->sp.out, c->h_st_cnts[2], cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    out->refs = c->cfg.by_ref && !iovec ? c->h_refs : nullptr;
    out->iov = iovec ? c->h_iov : nullptr;
    out->runs = c->h_run_status; out->n_runs = c->n_runs;
    out->msgs = c->h_msgs; out->n_msgs = n_msgs;
    out->resp = c->h_resp; out->resp_bytes = resp_bytes;
    return B2_OK;
}

// the running average message size, from which the next upload picks its tiles and pack kernel
static void note_avg_frame(b2_ctx* c, uint64_t bytes, uint32_t n_msgs) {
    if (n_msgs) { const uint32_t now = (uint32_t)(bytes / n_msgs); c->avg_frame = c->avg_frame ? (uint32_t)(((uint64_t)c->avg_frame * 3 + now) / 4) : now; }
}
extern "C" int b2_batch_download(b2_ctx* c, b2_batch_result* out) {
    if (!c || !out || !c->executed) { set_err("no executed batch"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    memset(out, 0, sizeof *out);
    if (c->small) {
        if (!c->small_copy_queued) CU(cudaMemcpyAsync(c->h_small, c->d_small, c->sm.total, cudaMemcpyDeviceToHost, c->stream));
        c->small_copy_queued = false;
        CU(cudaStreamSynchronize(c->stream));
        const uint32_t* tot = reinterpret_cast<const uint32_t*>(c->h_small);
        if (tot[2] & 3u) {
            // more messages / response bytes than the compact block holds: redo on the normal path
            c->small = false;
            int rc = launch_pipeline(c);
            if (rc != B2_OK) return rc;
            rc = download_normal(c, out);
            if (rc != B2_OK) return rc;
        } else {
            out->runs = reinterpret_cast<const b2_run_status*>(c->h_small + c->sm.off_rs); out->n_runs = c->n_runs;
            out->msgs = reinterpret_cast<const b2_msg_desc*>(c->h_small + c->sm.off_msgs); out->n_msgs = tot[0];
            out->resp = c->h_small + c->sm.off_resp; out->resp_bytes = tot[1];
            out->refs = c->cfg.by_ref ? reinterpret_cast<const b2_resp_ref*>(c->h_small + c->sm.off_refs) : nullptr;
            if (c->resp_mode == B2_RESP_IOVEC) refs_to_iov(c, out, c->host_bytes);
            if (c->stream_ran && c->h_st_cnts[2]) {          // multi-frame messages completed: their bytes follow
                CU(cudaMemcpyAsync(c->h_st_out, c->sp.out, c->h_st_cnts[2], cudaMemcpyDeviceToHost, c->stream));
                CU(cudaStreamSynchronize(c->stream));
            }
        }
    } else {
        int rc = download_normal(c, out);
        if (rc != B2_OK) return rc;
    }
    note_avg_frame(c, c->covered, out->n_msgs);
    out->kernel_ms = c->last_kernel_ms; out->n_launches = c->last_launches;
    c->stream_valid = c->stream_armed; c->stream_armed = false;
    return B2_OK;
}

extern "C" int b2_batch_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs) {
    int rc = b2_batch_upload(c, bytes, nbytes, runs, n_runs);
    if (rc != B2_OK) return rc;
    c->stream_armed = c->has_streams;
    rc = launch_pipeline(c);
    if (rc != B2_OK) return rc;
    c->executed = true;
    if (c->small) { CU(cudaMemcpyAsync(c->h_small, c->d_small, c->sm.total, cudaMemcpyDeviceToHost, c->stream)); c->small_copy_queued = true; }
    return B2_OK;
}

extern "C" int b2_batch_collect(b2_ctx* c, b2_batch_result* out) {
    int rc = b2_batch_download(c, out);
    if (rc != B2_OK) return rc;
    float ms = 0.f;
    if (c->n_stages) CU(cudaEventElapsedTime(&ms, c->ev[0], c->ev[c->n_stages]));
    c->last_kernel_ms = ms; out->kernel_ms = ms;
    return B2_OK;
}

extern "C" int b2_process_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                b2_batch_result* out) {
    int rc = b2_batch_submit(c, bytes, nbytes, runs, n_runs);
    if (rc != B2_OK) return rc;
    return b2_batch_collect(c, out);
}


// ---- the stream table (b2_stream_*) -------------------------------------------------------------------------------------------------
static void stream_free(b2_ctx* c) {
    for (void*& p : c->d_st_block) { cudaFree(p); p = nullptr; }
    for (void*& p : c->h_st_mapped) { cudaFreeHost(p); p = nullptr; }
    cudaFreeHost(c->h_st_cnts); c->h_st_cnts = nullptr; cudaFreeHost(c->h_st_out); c->h_st_out = nullptr;
    for (cudaEvent_t& e : c->st_ev) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (int i = 0; i < 4; i++) { cudaFree(c->d_sw[i]); c->d_sw[i] = nullptr; c->sw_have[i] = 0; }
    cudaFreeHost(c->h_sw_recs); c->h_sw_recs = nullptr; c->h_sw_have = 0; cudaFreeHost(c->h_sw_cnts); c->h_sw_cnts = nullptr;
    cudaFree(c->d_st_ring); c->d_st_ring = nullptr; cudaFree(c->d_swr); c->d_swr = nullptr;
    for (cudaEvent_t& e : c->sw_ev) if (e) { cudaEventDestroy(e); e = nullptr; }
    cudaGetLastError();
}
static int stream_configure(b2_ctx* c, uint32_t max_streams, uint32_t pending_bytes, uint32_t out_bytes);
extern "C" int b2_stream_configure(b2_ctx* c, uint32_t max_streams, uint32_t pending_bytes, uint32_t out_bytes) {
    const int rc = stream_configure(c, max_streams, pending_bytes, out_bytes);
    if (rc != B2_OK && c && !c->has_streams) stream_free(c);          // nothing of a failed attempt stays behind
    return rc;
}
static int stream_configure(b2_ctx* c, uint32_t max_streams, uint32_t pending_bytes, uint32_t out_bytes) {
    if (!c || max_streams == 0 || max_streams > (1u << 24) || pending_bytes == 0 || (pending_bytes & 15u)) { set_err("max_streams in 1 .. 2^24, pending_bytes a non-zero multiple of 16"); return B2_E_INVAL; }
    if (c->has_streams) { set_err("the stream table is already configured"); return B2_E_INVAL; }
    static_assert(sizeof(StreamEnt) == 80 && sizeof(b2_stream_msg) == 32 && sizeof(b2_stream_event) == 80 && sizeof(b2_stream_desc) == 32 && sizeof(b2_stream_state) == 32, "stream ABI layout");
    CU(cudaSetDevice(c->opt.device));
    CU(cudaStreamSynchronize(c->stream));
    ring_halt(c);
    StreamPass& S = c->sp;
    uint32_t cap = 16; while (cap < 2 * max_streams) cap <<= 1;
    const size_t mm = c->opt.max_msgs;
    S.cap = cap; S.pending_bytes = pending_bytes; S.out_cap = out_bytes ? out_bytes : c->opt.max_batch_bytes;
    const size_t dev_bytes[9] = { sizeof(StreamEnt) * (size_t)cap, (size_t)max_streams * pending_bytes, 4 * (16 + 2 * (size_t)cap), 4 * (size_t)cap, 4 * (size_t)cap,
                                  4 * mm, mm, 8 * mm, 64 * mm };
    for (int i = 0; i < 9; i++) if (cudaMalloc(&c->d_st_block[i], dev_bytes[i] + (i == 1 ? 16 : 0)) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the stream table failed"); return B2_E_NOMEM; }
    S.tab = (StreamEnt*)c->d_st_block[0]; S.pool = (uint8_t*)c->d_st_block[1]; S.cnts = (uint32_t*)c->d_st_block[2]; S.cnt = S.cnts + 16; S.fill = S.cnt + cap;
    S.base = (uint32_t*)c->d_st_block[3]; S.touched = (uint32_t*)c->d_st_block[4]; S.frame_slot = (uint32_t*)c->d_st_block[5]; S.rst = (uint8_t*)c->d_st_block[6];
    S.group = (uint32_t*)c->d_st_block[7]; S.tmp_msgs = (b2_stream_msg*)c->d_st_block[8];
    CU(cudaMemset(S.tab, 0, dev_bytes[0]));
    // results the kernels write in place: mapped host memory (msgs, events, control frames, per-run RST spans, the frame of close / set_connected)
    const size_t map_bytes[5] = { sizeof(b2_stream_msg) * mm, sizeof(b2_stream_event) * (size_t)max_streams, (size_t)kStreamCtrlMax * (mm + 2 * (size_t)max_streams), 8 * (size_t)c->opt.max_runs, 256 };
    void* dev[5];
    for (int i = 0; i < 5; i++) {
        if (cudaHostAlloc(&c->h_st_mapped[i], map_bytes[i], cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); set_err("cudaHostAlloc of the stream results failed"); return B2_E_NOMEM; }
        CU(cudaHostGetDevicePointer(&dev[i], c->h_st_mapped[i], 0));
    }
    c->h_st_msgs = (b2_stream_msg*)c->h_st_mapped[0]; c->h_st_events = (b2_stream_event*)c->h_st_mapped[1]; c->h_st_ctrl = (uint8_t*)c->h_st_mapped[2];
    c->h_st_run_ctrl = (uint32_t*)c->h_st_mapped[3]; c->h_st_ctl = (uint8_t*)c->h_st_mapped[4]; c->d_st_ctl = (uint8_t*)dev[4];
    S.msgs = (b2_stream_msg*)dev[0]; S.events = (b2_stream_event*)dev[1]; S.ctrl = (uint8_t*)dev[2]; S.run_ctrl = (uint32_t*)dev[3];
    if (cudaMalloc(&c->d_st_block[9], (size_t)S.out_cap + 16) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the stream out region failed"); return B2_E_NOMEM; }
    S.out = (uint8_t*)c->d_st_block[9];
    if (cudaHostAlloc((void**)&c->h_st_cnts, 64, cudaHostAllocDefault) != cudaSuccess || cudaHostAlloc((void**)&c->h_st_out, (size_t)S.out_cap + 16, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError(); set_err("cudaHostAlloc of the stream out mirror failed"); return B2_E_NOMEM;
    }
    memset(c->h_st_cnts, 0, 64);
    for (cudaEvent_t& e : c->st_ev) CU(cudaEventCreate(&e));
    c->st_max = max_streams; c->st_open = 0;
    c->st_keys.assign(cap, 0); c->st_state.assign(cap, 0); c->st_pool.assign(cap, 0);
    c->st_pool_free.clear(); for (uint32_t i = max_streams; i > 0; i--) c->st_pool_free.push_back(i - 1);
    c->has_streams = true;
    return B2_OK;
}

// a ring ticket of a context whose ring runs the stream pass is submitted and not collected: the table belongs to k_ring
static bool ring_owns_table(const b2_ctx* c) {
    if (!ring_runs_streams(c->ring_kind) || !ring_busy(c)) return false;
    set_err("a ring ticket is outstanding: b2_ring_wait it first, the stream table belongs to it");
    return true;
}

static uint32_t stream_find(const b2_ctx* c, int64_t id) {
    const uint32_t cap = c->sp.cap;
    uint32_t h = stream_hash((long long)id, cap);
    for (uint32_t k = 0; k < cap; k++, h = (h + 1) & (cap - 1)) {
        if (c->st_state[h] == 0) return kNone;
        if (c->st_state[h] == 1 && c->st_keys[h] == (long long)id) return h;
    }
    return kNone;
}

extern "C" int b2_stream_open(b2_ctx* c, const b2_stream_desc* streams, uint32_t n) {
    if (!c || !c->has_streams || (!streams && n)) { set_err("no stream table (b2_stream_configure) or null argument"); return B2_E_INVAL; }
    if (ring_owns_table(c)) return B2_E_INVAL;
    if (c->st_open + (uint64_t)n > c->st_max) { set_err("stream table full"); return B2_E_CAPACITY; }
    CU(cudaSetDevice(c->opt.device));
    CU(cudaStreamSynchronize(c->stream));
    // the slots are picked on the host mirror; the entries travel staged, contiguous slots in one copy each, one synchronisation for all
    const uint32_t cap = c->sp.cap;
    std::vector<std::pair<uint32_t, StreamEnt>> staged; staged.reserve(n);
    int rc = B2_OK;
    for (uint32_t i = 0; i < n && rc == B2_OK; i++) {
        const b2_stream_desc& d = streams[i];
        if (stream_find(c, d.stream_id) != kNone) { set_err("stream id is already open"); rc = B2_E_INVAL; break; }
        uint32_t h = stream_hash((long long)d.stream_id, cap);
        while (c->st_state[h] == 1) h = (h + 1) & (cap - 1);
        StreamEnt e; memset(&e, 0, sizeof e);
        e.id = d.stream_id; e.remote_id = d.remote_stream_id; e.host_socket = d.host_socket_id; e.max_buf = d.max_buf_size;
        e.flags = kStUsed | ((d.flags & B2_STREAM_CONNECTED) ? kStConnected : 0u) | ((d.flags & B2_STREAM_NEED_FEEDBACK) ? kStNeedFeedback : 0u);
        e.pool_idx = c->st_pool_free.back(); c->st_pool_free.pop_back();
        c->st_state[h] = 1; c->st_keys[h] = (long long)d.stream_id; c->st_pool[h] = e.pool_idx; c->st_open++;
        staged.push_back({ h, e });
    }
    std::sort(staged.begin(), staged.end(), [](const std::pair<uint32_t, StreamEnt>& a, const std::pair<uint32_t, StreamEnt>& b) { return a.first < b.first; });
    std::vector<StreamEnt> flat(staged.size());
    for (size_t i = 0; i < staged.size(); i++) flat[i] = staged[i].second;
    for (size_t i = 0; i < staged.size();) {
        size_t j = i + 1;
        while (j < staged.size() && staged[j].first == staged[j - 1].first + 1) j++;
        CU(cudaMemcpyAsync(c->sp.tab + staged[i].first, flat.data() + i, sizeof(StreamEnt) * (j - i), cudaMemcpyHostToDevice, c->stream));
        i = j;
    }
    CU(cudaStreamSynchronize(c->stream));
    return rc;
}

static int stream_ctl(b2_ctx* c, int64_t id, int op, int64_t remote, uint32_t flags, void* frame, uint32_t frame_cap, uint32_t* frame_len, uint32_t* slot_out) {
    if (!c || !c->has_streams || !frame_len || (!frame && frame_cap)) { set_err("no stream table (b2_stream_configure) or null argument"); return B2_E_INVAL; }
    if (frame_cap < kStreamCtrlMax) { set_err("frame_cap must be at least 64"); return B2_E_INVAL; }
    if (ring_owns_table(c)) return B2_E_INVAL;
    const uint32_t slot = stream_find(c, id);
    if (slot == kNone) { set_err("stream id is not open"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    uint32_t* d_len = reinterpret_cast<uint32_t*>(c->d_st_ctl + 128);
    k_stream_ctl<<<1, 1, 0, c->stream>>>(c->sp.tab, slot, op, (long long)remote, (flags & B2_STREAM_NEED_FEEDBACK) ? kStNeedFeedback : 0u, c->d_st_ctl, d_len);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    *frame_len = *reinterpret_cast<const uint32_t*>(c->h_st_ctl + 128);
    memcpy(frame, c->h_st_ctl, *frame_len);
    *slot_out = slot;
    return B2_OK;
}
extern "C" int b2_stream_set_connected(b2_ctx* c, int64_t stream_id, int64_t remote_stream_id, uint32_t flags, void* frame, uint32_t frame_cap, uint32_t* frame_len) {
    uint32_t slot;
    return stream_ctl(c, stream_id, 1, remote_stream_id, flags, frame, frame_cap, frame_len, &slot);
}
extern "C" int b2_stream_close(b2_ctx* c, int64_t stream_id, void* frame, uint32_t frame_cap, uint32_t* frame_len) {
    uint32_t slot;
    int rc = stream_ctl(c, stream_id, 0, 0, 0, frame, frame_cap, frame_len, &slot);
    if (rc != B2_OK) return rc;
    c->st_pool_free.push_back(c->st_pool[slot]); c->st_state[slot] = 2; c->st_open--;      // (a tombstone: probes for other ids walk over it)
    return B2_OK;
}
static int stream_read(b2_ctx* c, int64_t id, StreamEnt* e, uint32_t* slot) {
    if (!c || !c->has_streams) { set_err("no stream table (b2_stream_configure)"); return B2_E_INVAL; }
    *slot = stream_find(c, id);
    if (*slot == kNone) { set_err("stream id is not open"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(e, c->sp.tab + *slot, sizeof *e, cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_stream_query(b2_ctx* c, int64_t stream_id, b2_stream_state* out) {
    if (!out) { set_err("null argument"); return B2_E_INVAL; }
    StreamEnt e; uint32_t slot;
    int rc = stream_read(c, stream_id, &e, &slot); if (rc != B2_OK) return rc;
    out->local_consumed = e.local_consumed; out->remote_consumed = e.remote_consumed; out->pending_bytes = e.pending_len; out->error_code = e.error; out->reserved = 0;
    out->flags = ((e.flags & kStConnected) ? B2_STREAM_CONNECTED : 0u) | ((e.flags & kStNeedFeedback) ? B2_STREAM_NEED_FEEDBACK : 0u) |
                 ((e.flags & kStClosed) ? B2_STREAM_CLOSED : 0u) | ((e.flags & kStHandedOver) ? B2_STREAM_HANDED_OVER : 0u);
    return B2_OK;
}
extern "C" int b2_stream_take_pending(b2_ctx* c, int64_t stream_id, void* out, uint32_t cap, uint32_t* len) {
    if (!len || (!out && cap)) { set_err("null argument"); return B2_E_INVAL; }
    if (c && ring_owns_table(c)) return B2_E_INVAL;
    StreamEnt e; uint32_t slot;
    int rc = stream_read(c, stream_id, &e, &slot); if (rc != B2_OK) return rc;
    if (e.pending_len > cap) { set_err("the pending bytes do not fit"); return B2_E_CAPACITY; }
    if (e.pending_len) CU(cudaMemcpy(out, c->sp.pool + (size_t)e.pool_idx * c->sp.pending_bytes, e.pending_len, cudaMemcpyDeviceToHost));
    *len = e.pending_len;
    e.pending_len = 0; e.pending_frames = 0;
    CU(cudaMemcpy(c->sp.tab + slot, &e, sizeof e, cudaMemcpyHostToDevice));
    return B2_OK;
}
extern "C" int b2_stream_results(b2_ctx* c, b2_stream_batch_result* out) {
    if (!c || !out || !c->has_streams) { set_err("no stream table (b2_stream_configure) or null argument"); return B2_E_INVAL; }
    if (!c->stream_valid) { set_err("no collected batch of b2_process_batch / b2_batch_collect / b2_ring_wait"); return B2_E_INVAL; }
    memset(out, 0, sizeof *out);
    if (c->st_view_ticket) {                               // a ticket the ring served: the slot's stream section
        const uint8_t* slot = ring_slot(c, c->st_view_ticket), *sec = slot + c->ring_dev.off_st;
        const uint32_t* n = reinterpret_cast<const uint32_t*>(sec);
        out->msgs = reinterpret_cast<const b2_stream_msg*>(sec + kSecMsgs); out->n_msgs = n[0];
        out->events = reinterpret_cast<const b2_stream_event*>(sec + kSecEvents); out->n_events = n[1];
        out->out = sec + kSecOut; out->out_bytes = n[2]; out->ctrl = sec + kSecCtrl; out->ctrl_bytes = n[3];
        out->run_ctrl = reinterpret_cast<const uint32_t*>(sec + kSecRunCtrl); out->n_runs = reinterpret_cast<const RingSlotHdr*>(slot)->n_runs;
        return B2_OK;
    }
    if (!c->stream_ran) return B2_OK;                      // (a batch without runs)
    const uint32_t* n = c->h_st_cnts;
    out->msgs = c->h_st_msgs; out->n_msgs = n[0]; out->events = c->h_st_events; out->n_events = n[1];
    out->out = c->h_st_out; out->out_bytes = n[2]; out->ctrl = c->h_st_ctrl; out->ctrl_bytes = n[3];
    out->run_ctrl = c->h_st_run_ctrl; out->n_runs = c->n_runs;
    return B2_OK;
}

// ---- the sending side of a Stream (b2_stream_write, k_sw_*) ---------------------------------------------------------------------
// Staging of its own (never d_bytes / d_msgs / d_resp or the stream pass's results): the last batch's results and input bytes stay as
// they are, so FROM_MSG writes can read them in place.
static const char* const kSwStages[7] = { "stream_write_route", "stream_write_alloc", "stream_write_group", "stream_write_admit",
                                          "stream_write_scan", "stream_write_frames", "stream_write_copy" };
static int sw_reserve(b2_ctx* c, int i, size_t need) {          // device staging i holds at least `need` bytes (+ 32 of slack)
    if (need <= c->sw_have[i] && c->d_sw[i]) return B2_OK;
    size_t n = 4096; while (n < need) n <<= 1;
    cudaFree(c->d_sw[i]); c->d_sw[i] = nullptr; c->sw_have[i] = 0;
    if (cudaMalloc(&c->d_sw[i], n + 32) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the stream write staging failed"); return B2_E_NOMEM; }
    c->sw_have[i] = n;
    return B2_OK;
}
// the pinned host records hold at least n writes
static int sw_host_recs(b2_ctx* c, uint32_t n) {
    if ((size_t)n * sizeof(SwRec) <= c->h_sw_have) return B2_OK;
    cudaFreeHost(c->h_sw_recs); c->h_sw_recs = nullptr; c->h_sw_have = 0;
    size_t m = 4096; while (m < (size_t)n * sizeof(SwRec)) m <<= 1;
    if (cudaHostAlloc((void**)&c->h_sw_recs, m, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); set_err("cudaHostAlloc of the stream write records failed"); return B2_E_NOMEM; }
    c->h_sw_have = m;
    return B2_OK;
}
// Checks a write list and resolves it into recs[0, n) (b2_stream_write, b2_stream_ring_submit): a host-sourced payload at base + src_off
// of the nbytes the call carries; with from_msg a FROM_MSG write at the message of the last collected batch or ring ticket, else the flag
// is refused.  bound: the sum over writes of align16(len + ceil(len / seg) * 38), what the frames may take.  Nothing changes on failure.
static int sw_resolve(b2_ctx* c, const b2_stream_write_desc* writes, uint32_t n, uint32_t nbytes, uint64_t seg, const uint8_t* base,
                      bool from_msg, SwRec* recs, uint64_t& bound) {
    // FROM_MSG: the messages b2_stream_results describes — a ring ticket's only while it is the most recent one (the next ticket
    // overwrites the device input and the ring's out staging)
    const b2_stream_msg* from_msgs = c->h_st_msgs; const uint8_t* from_out = c->sp.out;
    uint32_t n_msgs = c->stream_valid && c->stream_ran ? c->h_st_cnts[0] : 0;
    if (from_msg && c->stream_valid && c->st_view_ticket) {
        b2_stream_batch_result v; b2_stream_results(c, &v);
        from_msgs = v.msgs; from_out = c->sp_ring.out; n_msgs = c->st_view_ticket + 1 == c->ring_next ? v.n_msgs : 0;
    }
    bound = 0;
    for (uint32_t i = 0; i < n; i++) {
        const b2_stream_write_desc& w = writes[i];
        SwRec& r = recs[i];
        r.id = w.stream_id; r.pad = 0;
        if (w.flags & ~B2_STREAM_W_FROM_MSG) { set_err("unknown b2_stream_write flag"); return B2_E_INVAL; }
        if (w.flags & B2_STREAM_W_FROM_MSG) {
            if (!from_msg) { set_err("B2_STREAM_W_FROM_MSG is refused in a ring ticket: the messages a ticket completes are not known when it is submitted (b2_stream_write between tickets)"); return B2_E_INVAL; }
            if (w.src_off >= n_msgs) { set_err("B2_STREAM_W_FROM_MSG: no such message in the last collected batch (or ring ticket, when it is the most recent)"); return B2_E_INVAL; }
            const b2_stream_msg& m = from_msgs[w.src_off];
            if ((m.flags & B2_STREAM_MSG_IN_INPUT) && !c->st_input) { set_err("B2_STREAM_W_FROM_MSG: a later call overwrote the last batch's input bytes on the device"); return B2_E_INVAL; }
            r.src = ((m.flags & B2_STREAM_MSG_IN_INPUT) ? c->st_input : from_out) + m.off; r.len = m.len;
        } else {
            if ((uint64_t)w.src_off + w.src_len > nbytes) { set_err("write outside bytes"); return B2_E_INVAL; }
            r.src = base + w.src_off; r.len = w.src_len;
        }
        const uint64_t nfr = r.len <= seg ? 1 : (r.len + seg - 1) / seg;
        bound += (r.len + nfr * kSwHeadMax + 15) & ~15ull;
    }
    return B2_OK;
}
// The grid path over the n records in h_sw_recs, whose host-sourced payloads point into d_sw[0]: bytes staged there, the seven k_sw_*
// kernels on the context's stream, the results and the used frame bytes copied to `results` / `out` (b2_stream_write, and the writes of
// a stream ring ticket whose runs overflowed).  bound: what sw_resolve computed.  *out_bytes: the frame bytes copied.
static int sw_launch(b2_ctx* c, const void* bytes, uint32_t nbytes, uint32_t n, uint64_t seg, uint64_t bound, b2_stream_write_result* results,
                     void* out, uint32_t* out_bytes) {
    int rc;
    const size_t cap = c->sp.cap;
    const size_t o_res = ((size_t)n * 24 + 15) & ~(size_t)15, o_slot = o_res + 32 * (size_t)n, o_group = o_slot + ((4 * (size_t)n + 15) & ~(size_t)15),
                 o_fb = o_group + 8 * (size_t)n, o_cb = o_fb + ((4 * (size_t)n + 15) & ~(size_t)15);
    if ((rc = sw_reserve(c, 1, bound)) != B2_OK || (rc = sw_reserve(c, 2, o_cb + 4 * (size_t)n)) != B2_OK || (rc = sw_reserve(c, 3, 64 + 16 * cap)) != B2_OK) return rc;
    if (!c->h_sw_cnts) {
        if (cudaHostAlloc((void**)&c->h_sw_cnts, 64, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); set_err("cudaHostAlloc failed"); return B2_E_NOMEM; }
        for (cudaEvent_t& e : c->sw_ev) CU(cudaEventCreate(&e));
    }
    uint8_t* blk = static_cast<uint8_t*>(c->d_sw[2]);
    uint32_t* per_slot = static_cast<uint32_t*>(c->d_sw[3]);
    SwPass P;
    P.tab = c->sp.tab; P.cap = c->sp.cap; P.recs = reinterpret_cast<const SwRec*>(blk); P.n = n; P.seg = (uint32_t)seg;
    P.cnts = per_slot; P.cnt = per_slot + 16; P.fill = P.cnt + cap; P.base = P.fill + cap; P.touched = P.base + cap;
    P.res = reinterpret_cast<b2_stream_write_result*>(blk + o_res); P.slot = reinterpret_cast<uint32_t*>(blk + o_slot); P.group = reinterpret_cast<uint32_t*>(blk + o_group);
    P.frame_base = reinterpret_cast<uint32_t*>(blk + o_fb); P.chunk_base = reinterpret_cast<uint32_t*>(blk + o_cb);
    P.out = static_cast<uint8_t*>(c->d_sw[1]);
    cudaStream_t s = c->stream;
    const uint32_t sms = c->n_sms, streams = n < c->st_max ? n : c->st_max;
    CU(cudaMemcpyAsync(blk, c->h_sw_recs, sizeof(SwRec) * (size_t)n, cudaMemcpyHostToDevice, s));
    if (nbytes) CU(cudaMemcpyAsync(c->d_sw[0], bytes, nbytes, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(per_slot, 0, 64 + 8 * cap, s));                 // counters | cnt | fill
    CU(cudaEventRecord(c->sw_ev[0], s));
    k_sw_route<<<grid(n, 256, sms * 4), 256, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[1], s));
    k_sw_alloc<<<grid(streams, 256, sms), 256, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[2], s));
    k_sw_group<<<grid(n, 256, sms * 4), 256, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[3], s));
    k_sw_admit<<<grid(streams, 4, sms * 8), 128, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[4], s));
    k_sw_scan<<<1, kSmallThreads, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[5], s));
    k_sw_frames<<<sms * 8, 256, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[6], s));
    k_sw_copy<<<sms * 8, 256, 0, s>>>(P); CU(cudaEventRecord(c->sw_ev[7], s));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(results, P.res, sizeof(b2_stream_write_result) * (size_t)n, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(c->h_sw_cnts, P.cnts, 64, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    c->sw_ran = true;
    *out_bytes = c->h_sw_cnts[2];
    if (c->h_sw_cnts[2]) {
        CU(cudaMemcpyAsync(out, P.out, c->h_sw_cnts[2], cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    return B2_OK;
}
extern "C" int b2_stream_write(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_stream_write_desc* writes, uint32_t n,
                               uint32_t max_segment_size, void* out, uint32_t out_cap, b2_stream_write_result* results) {
    static_assert(sizeof(b2_stream_write_desc) == 24 && sizeof(b2_stream_write_result) == 32 && sizeof(SwRec) == 24, "stream write ABI layout");
    if (!c || !c->has_streams || (!bytes && nbytes) || (!writes && n) || (!results && n) || (!out && out_cap)) { set_err("no stream table (b2_stream_configure) or null argument"); return B2_E_INVAL; }
    if (c->stream_armed) { set_err("a submitted batch must be collected first: the stream table belongs to it"); return B2_E_INVAL; }
    if (ring_owns_table(c) || ring_refuses(c, false)) return B2_E_INVAL;
    if (n > c->opt.max_msgs || nbytes > c->opt.max_batch_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    CU(cudaSetDevice(c->opt.device));
    const uint64_t seg = max_segment_size ? max_segment_size : 512ull << 20;       // -stream_write_max_segment_size (stream.cpp:39)
    int rc = sw_host_recs(c, n);
    if (rc == B2_OK) rc = sw_reserve(c, 0, nbytes);
    if (rc != B2_OK) return rc;
    // every argument is checked before anything changes; each record carries its payload's device address
    uint64_t bound = 0;
    if ((rc = sw_resolve(c, writes, n, nbytes, seg, static_cast<const uint8_t*>(c->d_sw[0]), true, c->h_sw_recs, bound)) != B2_OK) return rc;
    if (bound > out_cap || bound > c->opt.max_resp_bytes) { set_err("out_cap (or max_resp_bytes) below the sum of align16(len + ceil(len / seg) * 38)"); return B2_E_CAPACITY; }
    if (n == 0) return B2_OK;
    uint32_t used = 0;
    return sw_launch(c, bytes, nbytes, n, seg, bound, results, out, &used);
}

extern "C" int b2_stream_ring_enable(b2_ctx* c, uint32_t out_bytes) {
    if (!c || !c->has_streams) { set_err("no stream table (b2_stream_configure)"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::none) { set_err("b2_stream_ring_enable: once, before the context's first ring call"); return B2_E_INVAL; }
    if (out_bytes > (256u << 20)) { set_err("out_bytes above 256 MiB"); return B2_E_CAPACITY; }
    CU(cudaSetDevice(c->opt.device));
    CU(cudaStreamSynchronize(c->stream));
    if (cudaMalloc((void**)&c->d_st_ring, (size_t)kSecOut + ((out_bytes + 15u) & ~15u) + 16) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the ring's stream staging failed"); return B2_E_NOMEM; }
    CU(cudaMemset(c->sp.cnts, 0, 4 * (16 + 2 * (size_t)c->sp.cap)));         // counters | cnt | fill: the ring's tickets start from zeros
    StreamPass R = c->sp;                   // table, pool and scratch shared with the batch calls; results and counters its own
    R.cnts = reinterpret_cast<uint32_t*>(c->d_st_ring);
    R.events = reinterpret_cast<b2_stream_event*>(c->d_st_ring + kSecEvents); R.msgs = reinterpret_cast<b2_stream_msg*>(c->d_st_ring + kSecMsgs);
    R.ctrl = c->d_st_ring + kSecCtrl; R.run_ctrl = reinterpret_cast<uint32_t*>(c->d_st_ring + kSecRunCtrl);
    R.out = c->d_st_ring + kSecOut; R.out_cap = out_bytes;
    c->sp_ring = R; c->ring_kind = RingKind::batch_streams;
    return B2_OK;
}

// ---- the persistent latency path: submit ring + the resident kernel of the context's ring kind ------------------------------------
static void ring_halt(b2_ctx* c) {
    if (!c->ring_ctl) return;
    c->ring_ctl[0] = 1; __sync_synchronize();
    cudaStreamSynchronize(c->ring_stream);
    c->ring_ctl[0] = 0; c->ring_ctl[1] = 0; __sync_synchronize();
}
static H2RingDev h2_ring_dev(const b2_ctx* c);
static H2ClientRingDev h2_client_ring_dev(const b2_ctx* c);
// (re)launches the resident kernel of the context's ring kind on ring_stream
static int ring_launch(b2_ctx* c) {
    RingDev R = c->ring_dev;                // (the slot parts)
    R.slots = c->ring_slots; R.slot_stride = c->ring_stride; R.ctl = c->ring_ctl; R.next_ticket = c->d_ring_ticket;
    unsigned long long idle_ms = 20; if (const char* e = getenv("B2_RING_IDLE_MS")) idle_ms = (unsigned long long)atoi(e);
    R.idle_ns = idle_ms * 1000000ull;
    R.d_bytes = c->d_bytes; R.d_meta = c->d_meta; R.d_small = c->d_small;
    c->ring_ctl[1] = 1; __sync_synchronize();
    switch (c->ring_kind) {
    case RingKind::h2_server: {             // k_h2_ring<true> on a turn-enabled context (b2_h2_ring_turn_enable)
        const H2RingDev H = h2_ring_dev(c);
        if (c->h2r_max_resps) k_h2_ring<true><<<1, kSmallThreads, kH2RingSmem, c->ring_stream>>>(R, H, c->h2t_dev);
        else k_h2_ring<false><<<1, kSmallThreads, kH2RingSmem, c->ring_stream>>>(R, H, H2TurnDev{});
        break;
    }
    case RingKind::h2_client: { const H2ClientRingDev H = h2_client_ring_dev(c); k_h2_client_ring<<<1, kSmallThreads, kH2ClientRingSmem, c->ring_stream>>>(R, H); break; }
    default: {                              // batch, batch_streams, batch_stream_writes, batch_client, batch_replies
        const bool was_small = c->small; c->small = false;
        BatchPtrs B = make_ptrs(c);
        c->small = was_small;
        B.bytes = c->d_bytes;
        const StreamPass SP = ring_runs_streams(c->ring_kind) ? c->sp_ring : StreamPass{};   // (tab null: the ring runs no stream pass)
        if (ring_packs(c->ring_kind)) {
            // the scratch of b2_pack_requests / b2_pack_responses, except that the records and their offsets go to d_msgs / d_refs, which
            // k_ring leaves alone
            PackRingDev Q = c->pr_dev;
            Q.recs = reinterpret_cast<uint8_t*>(c->d_msgs); Q.offs = reinterpret_cast<uint32_t*>(c->d_refs); Q.lens = Q.offs + c->opt.max_msgs;
            Q.scratch = c->d_unz; Q.out = c->d_resp;
            if (c->ring_kind == RingKind::batch_client) k_ring<RingBody::requests><<<1, kSmallThreads, sizeof(SmallSmem), c->ring_stream>>>(R, B, c->cfg, SP, Q);
            else k_ring<RingBody::replies><<<1, kSmallThreads, sizeof(SmallSmem), c->ring_stream>>>(R, B, c->cfg, SP, Q);
        } else if (c->ring_kind == RingKind::batch_stream_writes) {
            k_ring<RingBody::stream_writes><<<1, kSmallThreads, sizeof(SmallSmem), c->ring_stream>>>(R, B, c->cfg, SP, c->swr_dev);
        } else k_ring<RingBody::batch><<<1, kSmallThreads, sizeof(SmallSmem), c->ring_stream>>>(R, B, c->cfg, SP, PackRingDev{});
    }
    }
    c->ring_launches++;
    CU(cudaGetLastError());
    return B2_OK;
}
// the kRingSlots slots of `end` bytes each (pinned + mapped), the control words, the ticket counter and the ring stream: once per context,
// for whichever resident kernel it runs
static int ring_alloc(b2_ctx* c, uint64_t end) {
    if (end > (1ull << 31)) { set_err("ring slot too large: lower the capacities"); return B2_E_CAPACITY; }
    c->ring_stride = (uint32_t)((end + 4095u) & ~4095ull);
    CU(cudaHostAlloc((void**)&c->ring_slots, (size_t)c->ring_stride * kRingSlots, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(c->ring_slots, 0, (size_t)c->ring_stride * kRingSlots);
    CU(cudaHostAlloc((void**)&c->ring_ctl, 64, cudaHostAllocMapped | cudaHostAllocPortable));
    memset((void*)c->ring_ctl, 0, 64);
    CU(cudaMalloc((void**)&c->d_ring_ticket, 8));
    const uint32_t init[2] = { 1, 0 }; CU(cudaMemcpy(c->d_ring_ticket, init, 8, cudaMemcpyHostToDevice));
    CU(cudaStreamCreateWithFlags(&c->ring_stream, cudaStreamNonBlocking));
    return B2_OK;
}
extern "C" int b2_ring_start(b2_ctx* c) {
    if (!c) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    if (c->ring_kind == RingKind::none) c->ring_kind = RingKind::batch;
    if (!c->ring_slots) {                   // k_ring's slot (the h2 kinds lay out theirs when enabled): [header | runs | staged input | output block | stream section]
        SlotLayout L;
        RingDev& R = c->ring_dev;
        R.off_runs = L.add(kSmallRuns * sizeof(b2_run));
        R.off_in = L.add(kSmallBytes + 1024u);
        R.off_out = L.add(kSmallBlock);
        if (c->ring_kind == RingKind::batch_streams) R.off_st = L.add(kSecOut + ((c->sp_ring.out_cap + 15u) & ~15u));
        int rc = ring_alloc(c, L.end); if (rc != B2_OK) return rc;
        CU(cudaFuncSetAttribute(k_ring<RingBody::batch>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallSmem)));
    }
    if (!c->ring_ctl[1]) return ring_launch(c);
    return B2_OK;
}
// the batch bytes as the kernel pulls them: in place when they already live in pinned + mapped memory (b2_block_alloc), else staged into
// the slot's off_in
static unsigned long long ring_stage(b2_ctx* c, uint8_t* slot, const void* bytes, uint32_t nbytes) {
    unsigned long long dev = 0;
    if (bytes == c->ring_pin_base) dev = c->ring_pin_dev;
    else {
        cudaPointerAttributes at; memset(&at, 0, sizeof at);
        if (cudaPointerGetAttributes(&at, bytes) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) {
            dev = (unsigned long long)(uintptr_t)at.devicePointer; c->ring_pin_base = bytes; c->ring_pin_dev = dev;
        } else cudaGetLastError();
    }
    if (!dev) { memcpy(slot + c->ring_dev.off_in, bytes, nbytes); dev = (unsigned long long)(uintptr_t)(slot + c->ring_dev.off_in); }
    return dev;
}
// A submission in three steps, each kind's own parts in between.  ring_claim: the slot of the next ticket, or null when the ring is full
// (wait_call: what frees a slot).  ring_fill: what every ticket carries — the batch bytes, the runs and their sizes in the header; the
// resident kernel pulls them into d_bytes / d_meta and serves the ticket over the batch scratch.  ring_ring: the doorbell.
static uint8_t* ring_claim(b2_ctx* c, const char* wait_call) {
    if (!c->ring_collected[c->ring_next % kRingSlots]) { set_err("submit ring full: %s the oldest ticket first", wait_call); return nullptr; }
    return ring_slot(c, c->ring_next);
}
static RingSlotHdr* ring_fill(b2_ctx* c, uint8_t* slot, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs) {
    overwrites(c, kDevInput | kDevBatch);
    RingSlotHdr* h = reinterpret_cast<RingSlotHdr*>(slot);
    h->bytes_dev = ring_stage(c, slot, bytes, nbytes);
    if (n_runs) memcpy(slot + c->ring_dev.off_runs, runs, sizeof(b2_run) * (size_t)n_runs);
    h->n_runs = n_runs; h->nbytes = nbytes;
    return h;
}
// k_ring's compact output block of the ticket (small_layout), in its header
static void ring_compact(const b2_ctx* c, RingSlotHdr* h, const SmallLayout& L) {
    h->small_msgs = L.msgs; h->small_resp = L.resp; h->off_rs = L.off_rs; h->off_msgs = L.off_msgs;
    h->off_refs = L.off_refs; h->off_resp = L.off_resp; h->total = L.total; h->by_ref = c->cfg.by_ref;
}
// marks the next ticket outstanding, rings its doorbell (everything else the host stores in the slot first) and relaunches the kernel if it
// idled out
static int ring_ring(b2_ctx* c, RingSlotHdr* h, const void* bytes, uint32_t* ticket) {
    const uint32_t t = c->ring_next;
    c->ring_bytes[t % kRingSlots] = bytes; c->ring_collected[t % kRingSlots] = false;
    __sync_synchronize();
    h->submit = t;
    __sync_synchronize();
    c->ring_next = t + 1;
    *ticket = t;
    if (!c->ring_ctl[1]) { CU(cudaSetDevice(c->opt.device)); return ring_launch(c); }   // the kernel idled out (or was never started)
    return B2_OK;
}
// spins until the kernel released `ticket`; starts the kernel again when it lost the exit race with the submission
static int ring_spin(b2_ctx* c, const RingSlotHdr* h, uint32_t ticket) {
    uint64_t spins = 0;
    while (h->done != ticket) {
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
        if ((++spins & 0xfffff) == 0) {
            if (!c->ring_ctl[1]) { CU(cudaSetDevice(c->opt.device)); int rc = ring_launch(c); if (rc != B2_OK) return rc; }   // lost the exit race: start it again
            if (cudaStreamQuery(c->ring_stream) != cudaErrorNotReady && h->done != ticket && !c->ring_ctl[1]) continue;
            if (spins > (1ull << 34)) { set_err("ring kernel did not answer"); return B2_E_CUDA; }
        }
    }
    __sync_synchronize();
    return B2_OK;
}
// The slot of `ticket` once the kernel released it, marked collected; else null, with the error set and rc the code.  args_ok: the
// caller's own checks (bad_ticket: its text for them and for a ticket that is not outstanding).  A context whose ring runs the stream
// pass collects in ticket order.
static uint8_t* ring_collect(b2_ctx* c, bool args_ok, uint32_t ticket, const char* bad_ticket, int& rc) {
    rc = B2_E_INVAL;
    if (!args_ok || !c->ring_slots || ticket == 0 || ticket >= c->ring_next || ticket + kRingSlots < c->ring_next) { set_err(bad_ticket); return nullptr; }
    if (c->ring_collected[ticket % kRingSlots]) { set_err("ticket already collected"); return nullptr; }
    const bool in_order = ring_runs_streams(c->ring_kind);
    if (in_order && ticket != c->ring_next_wait) { set_err("a context whose ring runs the stream pass collects its tickets in ticket order"); return nullptr; }
    uint8_t* slot = ring_slot(c, ticket);
    if ((rc = ring_spin(c, reinterpret_cast<const RingSlotHdr*>(slot), ticket)) != B2_OK) return nullptr;
    c->ring_collected[ticket % kRingSlots] = true;
    if (in_order) c->ring_next_wait = ticket + 1;
    return slot;
}
static int ring_batch_result(b2_ctx* c, uint32_t ticket, uint8_t* slot, b2_batch_result* out, bool unpark = true);
extern "C" int b2_ring_stop(b2_ctx* c) { if (!c) return B2_E_INVAL; cudaSetDevice(c->opt.device); ring_halt(c); return B2_OK; }

extern "C" int b2_ring_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t* ticket) {
    if (!c || !bytes || !runs || !ticket || n_runs == 0) { set_err("null argument"); return B2_E_INVAL; }
    if (c->has_streams && !ring_runs_streams(c->ring_kind)) { set_err("the ring path runs the stream pass only after b2_stream_ring_enable: use b2_batch_submit on a context with a stream table"); return B2_E_INVAL; }
    if (c->ring_kind == RingKind::h2_server) { set_err("this context's ring serves h2 (b2_h2_ring_enable): use b2_h2_ring_submit"); return B2_E_INVAL; }
    if (c->ring_kind == RingKind::h2_client) { set_err("this context's ring serves h2 client connections (b2_h2_client_ring_enable): use b2_h2_client_ring_submit"); return B2_E_INVAL; }
    if (c->ring_kind == RingKind::batch_client) { set_err("this context's ring serves client turns (b2_client_ring_enable): use b2_client_ring_submit"); return B2_E_INVAL; }
    if (c->ring_kind == RingKind::batch_replies) { set_err("this context's ring serves server turns (b2_ring_turn_enable): use b2_ring_turn_submit"); return B2_E_INVAL; }
    if (c->ring_kind == RingKind::batch_stream_writes) { set_err("this context's ring serves Stream producer turns (b2_stream_ring_write_enable): use b2_stream_ring_submit"); return B2_E_INVAL; }
    if (nbytes > kSmallBytes || n_runs > kSmallRuns) { set_err("b2_ring_submit serves batches up to 128 KiB / 512 runs: use b2_batch_submit"); return B2_E_CAPACITY; }
    if (!c->ring_slots) { int rc = b2_ring_start(c); if (rc != B2_OK) return rc; }
    uint8_t* slot = ring_claim(c, "b2_ring_wait");
    if (!slot) return B2_E_CAPACITY;
    for (uint32_t r = 0; r < n_runs; r++)
        if ((runs[r].offset & 15u) || (uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run offset must be 16-aligned and inside the batch"); return B2_E_INVAL; }
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    ring_compact(c, h, small_layout(nbytes, n_runs, c->opt.max_msgs));
    return ring_ring(c, h, bytes, ticket);
}

extern "C" int b2_ring_wait(b2_ctx* c, uint32_t ticket, b2_batch_result* out) {
    if (c && c->ring_kind == RingKind::h2_server) { set_err("this context's ring serves h2: use b2_h2_ring_wait"); return B2_E_INVAL; }
    if (c && c->ring_kind == RingKind::h2_client) { set_err("this context's ring serves h2 client connections: use b2_h2_client_ring_wait"); return B2_E_INVAL; }
    if (c && c->ring_kind == RingKind::batch_client) { set_err("this context's ring serves client turns: use b2_client_ring_wait"); return B2_E_INVAL; }
    if (c && c->ring_kind == RingKind::batch_replies) { set_err("this context's ring serves server turns: use b2_ring_turn_wait"); return B2_E_INVAL; }
    if (c && c->ring_kind == RingKind::batch_stream_writes) { set_err("this context's ring serves Stream producer turns: use b2_stream_ring_wait"); return B2_E_INVAL; }
    int rc;
    uint8_t* slot = ring_collect(c, c && out, ticket, "bad ring ticket", rc);
    if (!slot) return rc;
    return ring_batch_result(c, ticket, slot, out);
}
// The runs' result of a collected k_ring ticket, from its compact block, or from the big pipeline when the runs overflowed it.  unpark:
// release the kernel parked behind an overflowing ticket of a stream ring here (false: the caller has more of the ticket to serve first,
// and releases it with ring_unpark)
static void ring_unpark(b2_ctx* c, uint32_t ticket) { __sync_synchronize(); c->ring_ctl[3] = ticket; __sync_synchronize(); }
static int ring_batch_result(b2_ctx* c, uint32_t ticket, uint8_t* slot, b2_batch_result* out, bool unpark) {
    int rc;
    const uint32_t si = ticket % kRingSlots;
    const bool streams = ring_runs_streams(c->ring_kind);
    RingSlotHdr* h = reinterpret_cast<RingSlotHdr*>(slot);
    memset(out, 0, sizeof *out);
    const uint8_t* ob = slot + c->ring_dev.off_out;
    const uint32_t* tot = reinterpret_cast<const uint32_t*>(ob);
    if (tot[2] & 3u) {
        // more messages / reply bytes than the compact block holds: the big pipeline serves the ticket.  With the stream pass on the ring,
        // k_ring ran no pass for it (the pipeline runs its own) and parks before the next one's pull until ctl[3] releases it, so that the
        // table sees the tickets in ticket order; otherwise the ring must be quiet first
        if (!streams && ring_busy(c)) { set_err("ring overflow fallback needs the other tickets collected first"); return B2_E_CAPACITY; }
        if (!streams) ring_halt(c);
        const bool allow = c->allow_small; c->allow_small = false;
        rc = b2_process_batch(c, c->ring_bytes[si], h->nbytes, reinterpret_cast<const b2_run*>(slot + c->ring_dev.off_runs), h->n_runs, out);
        c->allow_small = allow;
        if (streams && unpark) ring_unpark(c, ticket);
        return rc;
    }
    out->runs = reinterpret_cast<const b2_run_status*>(ob + h->off_rs); out->n_runs = h->n_runs;
    out->msgs = reinterpret_cast<const b2_msg_desc*>(ob + h->off_msgs); out->n_msgs = tot[0];
    out->resp = ob + h->off_resp; out->resp_bytes = tot[1];
    out->refs = h->by_ref ? reinterpret_cast<const b2_resp_ref*>(ob + h->off_refs) : nullptr;
    if (c->resp_mode == B2_RESP_IOVEC) refs_to_iov(c, out, c->ring_bytes[si]);
    out->n_launches = 0; out->kernel_ms = 0.f;
    if (streams) { c->stream_valid = true; c->st_view_ticket = ticket; c->st_input = c->d_bytes; }
    note_avg_frame(c, h->nbytes, out->n_msgs);
    return B2_OK;
}
extern "C" uint64_t b2_ring_launches(b2_ctx* c) { return c ? c->ring_launches : 0; }
// device-side phase times of a collected ticket, ns since the kernel saw the doorbell: [0] header read [1] runs + bytes pulled [2] cut / decode / pack done [3] results pushed
extern "C" int b2_ring_phase_ns(b2_ctx* c, uint32_t ticket, uint64_t out[4]) {
    if (!c || !c->ring_slots || !out) return B2_E_INVAL;
    const RingSlotHdr* h = reinterpret_cast<const RingSlotHdr*>(ring_slot(c, ticket));
    for (int k = 0; k < 4; k++) out[k] = h->stamps[k + 1] - h->stamps[0];
    return B2_OK;
}

// measurement helper: wall-clock microseconds of `iters` back-to-back calls, one batch each, timed inside the library so that
// the caller's language runtime is not part of the number (bench.py's latency line)
extern "C" int b2_latency_probe(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t iters, int use_ring, float* us_out) {
    if (!c || !us_out) return B2_E_INVAL;
    b2_batch_result res;
    for (uint32_t i = 0; i < iters; i++) {
        timespec t0, t1; clock_gettime(CLOCK_MONOTONIC, &t0);
        int rc;
        if (use_ring) { uint32_t t = 0; rc = b2_ring_submit(c, bytes, nbytes, runs, n_runs, &t); if (rc == B2_OK) rc = b2_ring_wait(c, t, &res); }
        else rc = b2_process_batch(c, bytes, nbytes, runs, n_runs, &res);
        clock_gettime(CLOCK_MONOTONIC, &t1);
        if (rc != B2_OK) return rc;
        if (res.n_msgs == 0) { set_err("latency probe batch produced no messages"); return B2_E_INVAL; }
        us_out[i] = (float)((t1.tv_sec - t0.tv_sec) * 1e6 + (t1.tv_nsec - t0.tv_nsec) * 1e-3);
    }
    return B2_OK;
}

extern "C" int b2_stage_times(b2_ctx* c, const char** names, float* ms, int cap) {
    if (!c) return B2_E_INVAL;
    int n = c->n_stages < cap ? c->n_stages : cap;
    for (int i = 0; i < n; i++) {
        names[i] = c->stage_names[i];
        float t = 0.f;
        cudaEventElapsedTime(&t, c->ev[i], c->ev[i + 1]);
        ms[i] = t;
    }
    int total = c->n_stages;
    if (c->stream_valid && c->stream_ran) {          // the stream pass of the last collected batch, kernel by kernel
        for (int i = 0; i < 5; i++, total++) if (total < cap) { names[total] = kStreamStages[i]; float t = 0.f; cudaEventElapsedTime(&t, c->st_ev[i], c->st_ev[i + 1]); ms[total] = t; }
    }
    if (c->sw_ran) {                                 // the last b2_stream_write, kernel by kernel
        for (int i = 0; i < 7; i++, total++) if (total < cap) { names[total] = kSwStages[i]; float t = 0.f; cudaEventElapsedTime(&t, c->sw_ev[i], c->sw_ev[i + 1]); ms[total] = t; }
    }
    return total;
}

// what the last upload / launch decided: [0] tile bytes [1] tiles [2] frame offsets kept per tile [3] 1 = the fused kernel served it
extern "C" int b2_set_walk_group(b2_ctx* c, uint32_t mode) {
    if (!c || mode > 8) { set_err("walk group mode: 0 auto, 1 off, 2..8 tiles per group"); return B2_E_INVAL; }
    c->walk_group_mode = mode;
    overwrites(c, kDevBatch);                       // (the uploaded batch's groups were laid out for the old mode)
    return B2_OK;
}

extern "C" int b2_walk_group(b2_ctx* c) { return c ? (int)c->walk_group_last : B2_E_INVAL; }

extern "C" int b2_batch_info(b2_ctx* c, uint32_t out[4]) {
    if (!c || !out) return B2_E_INVAL;
    out[0] = c->cfg.tile_bytes; out[1] = c->n_tiles; out[2] = c->cfg.spec_k; out[3] = c->fused_last ? 1u : 0u;
    return B2_OK;
}

// Registers are allocated per warp in units of 256 (8 per thread); shared memory per block adds the SM's per-block reserve.  An SM's
// shared memory is configured in steps (sm_90: 0, 8, 16, 32, 64, 100, 132, 164, 196 or 228 KB): one that a k_fused CTA holds is set to
// the smallest step that holds the CTA, and the blocks beside it share what that step leaves (a k_resolve block with its tile records in
// shared memory was seen to wait for the k_fused CTA to end).
static uint32_t block_regs(const b2_resident_kernel& k) { return (k.threads + 31) / 32 * ((k.regs * 32 + 255) / 256 * 256); }
static uint32_t smem_step(uint32_t bytes, uint32_t most) {
    static const uint32_t kKB[] = { 0, 8, 16, 32, 64, 100, 132, 164, 196, 228 };
    for (uint32_t kb : kKB) if (kb * 1024 >= bytes) return std::min(kb * 1024, most);
    return most;
}
extern "C" int b2_resident_plan(b2_ctx* c, b2_resident_kernel* out, int cap) {
    if (!c || (!out && cap > 0)) { set_err("null argument"); return B2_E_INVAL; }
    if (!c->plan[kPlanFused].name) { set_err("this build has no function attributes to plan with"); return B2_E_INVAL; }
    b2_resident_kernel k[kPlanKernels];
    memcpy(k, c->plan, sizeof k);
    const uint32_t fw = fused_warps(c);
    k[kPlanFused].threads = fw * 32; k[kPlanFused].smem_bytes += (uint32_t)(sizeof(FusedWarpSmem) * fw);
    k[kPlanResolve].smem_bytes += (uint32_t)resolve_smem(c, true);
    if (c->walk_group > 1) k[kPlanWalk].threads = kWalkGroupThreads;
    // the room one k_fused CTA leaves on its SM
    const b2_resident_kernel& f = k[kPlanFused];
    const uint32_t f_regs = block_regs(f), f_smem = f.smem_bytes + c->block_smem_reserve;
    const uint32_t room_regs = c->sm_regs > f_regs ? c->sm_regs - f_regs : 0, f_step = smem_step(f_smem, c->sm_smem);
    const uint32_t room_smem = f_step > f_smem ? f_step - f_smem : 0;
    const uint32_t room_warps = c->sm_warps > fw ? c->sm_warps - fw : 0, room_blocks = c->sm_blocks > 1 ? c->sm_blocks - 1 : 0;
    for (int i = 0; i < kPlanKernels; i++) {
        uint32_t n = room_blocks;
        n = std::min(n, room_regs / std::max(1u, block_regs(k[i])));
        n = std::min(n, room_smem / (k[i].smem_bytes + c->block_smem_reserve));
        n = std::min(n, room_warps / ((k[i].threads + 31) / 32));
        k[i].fits = n;
    }
    for (int i = 0; i < kPlanKernels && i < cap; i++) out[i] = k[i];
    return kPlanKernels;
}

extern "C" int b2_device_pci_bus_id(int device, char* out, int cap) {
    if (!out || cap < 13) return B2_E_INVAL;
    if (cudaDeviceGetPCIBusId(out, cap, device) != cudaSuccess) { cudaGetLastError(); return B2_E_CUDA; }
    return B2_OK;
}

extern "C" int b2_counters_read(b2_ctx* c, int64_t out[B2_N_COUNTERS]) {
    if (!c || !out) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    CU(cudaMemcpy(out, c->d_counters, 8 * B2_N_COUNTERS, cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" void* b2_counters_device_ptr(b2_ctx* c) { return c ? (void*)c->d_counters : nullptr; }
// ncclAllReduce(sendbuff, recvbuff, count, ncclInt64 = 4, ncclSum = 0, comm, stream) — nccl.h; looked up in the process, not linked
extern "C" int b2_counters_allreduce(b2_ctx* c, void* nccl_comm) {
    if (!c || !nccl_comm) { set_err("null argument"); return B2_E_INVAL; }
    typedef int (*allreduce_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
    static allreduce_fn fn = reinterpret_cast<allreduce_fn>(dlsym(RTLD_DEFAULT, "ncclAllReduce"));
    if (!fn) { set_err("ncclAllReduce is not loaded in this process"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    const int rc = fn(c->d_counters, c->d_counters, B2_N_COUNTERS, 4 /*ncclInt64*/, 0 /*ncclSum*/, nccl_comm, c->stream);
    if (rc != 0) { char code[16]; snprintf(code, sizeof code, "%d", rc); set_err("ncclAllReduce failed: ncclResult_t %s", code); return B2_E_CUDA; }
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// device pointers of the resident batch, for harnesses that time or inspect kernels directly
extern "C" void* b2_debug_resp_device_ptr(b2_ctx* c) { return c ? (void*)c->d_resp : nullptr; }

__global__ void k_crc32c_batch(const uint8_t* bytes, const uint32_t* offs, const uint32_t* lens, uint32_t n, uint32_t* out,
                               const uint32_t* adv, uint32_t init_crc = 0) {
    __shared__ uint32_t s_hot[kCrcHotWords];
    crc_tabs_to_smem(s_hot, adv);
    CrcTabs ct; ct.hot = s_hot; ct.tree = adv + kCrcHotWords;
    const uint32_t lane = threadIdx.x & 31, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += n_warps) {
        const uint32_t c = warp_crc32c_update(init_crc ^ 0xffffffffu, bytes + offs[i], lens[i], lane, ct) ^ 0xffffffffu;   // Extend(init_crc, ...)
        if (lane == 0) out[i] = c;
    }
}

// the outputs of a batch call lie back to back in `out`, 16-byte aligned: the next one, `need` bytes, at *off; false once past out_cap
static bool out_place(uint64_t& total, uint64_t need, uint32_t out_cap, uint32_t* off) { *off = (uint32_t)total; total += (need + 15) & ~15ull; return total <= out_cap; }
extern "C" int b2_crc32c_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const uint32_t* offs, const uint32_t* lens,
                               uint32_t n, uint32_t* out) {
    if (!c || !bytes || !offs || !lens || !out) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    if (nbytes > c->opt.max_batch_bytes || n > c->opt.max_msgs) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    for (uint32_t i = 0; i < n; i++) if ((uint64_t)offs[i] + lens[i] > nbytes) { set_err("slice outside buffer"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_frame_off, offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_slot, lens, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    if (n) k_crc32c_batch<<<c->n_sms * 8, 256, 0, c->stream>>>(c->d_bytes, c->d_frame_off, c->d_slot, n, (uint32_t*)c->d_aux, c->d_crc_adv);
    CU(cudaMemcpyAsync(out, c->d_aux, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

__global__ void k_snappy_batch(const uint8_t* bytes, const uint32_t* offs, const uint32_t* lens, uint32_t n, uint8_t* out,
                               const uint32_t* out_offs, const uint32_t* out_caps, int32_t* out_lens) {
    const uint32_t lane = threadIdx.x & 31, n_warps = (gridDim.x * blockDim.x) >> 5;
    __shared__ __align__(16) uint8_t s_rings[8 * kSnapRing];
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += n_warps) {
        uint32_t produced = 0;
        const bool ok = out_caps[i] != 0xffffffffu &&
                        warp_snappy_decode(bytes + offs[i], lens[i], out + out_offs[i], out_caps[i], lane, produced, s_rings + (threadIdx.x >> 5) * kSnapRing);
        if (lane == 0) out_lens[i] = ok ? (int32_t)produced : -1;
    }
}

extern "C" int b2_snappy_uncompress_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const uint32_t* offs, const uint32_t* lens,
                                          uint32_t n, void* out, uint32_t out_cap, uint32_t* out_offs, int32_t* out_lens) {
    if (!c || !bytes || !offs || !lens || !out || !out_offs || !out_lens) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    if (nbytes > c->opt.max_batch_bytes || n > c->opt.max_msgs || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    // output layout from the announced lengths (the preamble varint), nothing else is read on the host
    std::vector<uint32_t> caps(n);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        if ((uint64_t)offs[i] + lens[i] > nbytes) { set_err("slice outside buffer"); return B2_E_INVAL; }
        const uint8_t* p = (const uint8_t*)bytes + offs[i];
        uint32_t v = 0, shift = 0, k = 0; bool ok = false;
        while (k < lens[i] && shift < 32) { const uint32_t b = p[k++]; v |= (b & 0x7f) << shift; if (b < 128) { ok = true; break; } shift += 7; }
        const bool valid = ok && (uint64_t)v <= 32ull * lens[i] + 64ull;       // else it cannot be a valid stream: no output
        caps[i] = valid ? v : 0xffffffffu;
        if (!out_place(total, valid ? v : 0, out_cap, &out_offs[i])) { set_err("output exceeds out_cap"); return B2_E_CAPACITY; }
    }
    CU(cudaSetDevice(c->opt.device));
    uint32_t* d_offs = c->d_frame_off; uint32_t* d_lens = c->d_slot; uint32_t* d_ooffs = c->d_frame_run;
    uint32_t* d_caps = (uint32_t*)c->d_jobs; int32_t* d_olens = (int32_t*)c->d_aux;
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_offs, offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_lens, lens, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_ooffs, out_offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_caps, caps.data(), 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    if (n) k_snappy_batch<<<c->n_sms * 4, 256, 0, c->stream>>>(c->d_bytes, d_offs, d_lens, n, c->d_unz, d_ooffs, d_caps, d_olens);
    CU(cudaMemcpyAsync(out_lens, d_olens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    if (total) CU(cudaMemcpyAsync(out, c->d_unz, total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

__global__ void __launch_bounds__(256) k_snappy_compress_batch(const uint8_t* bytes, const uint32_t* offs, const uint32_t* lens, uint32_t n,
                                                               uint8_t* out, const uint32_t* out_offs, uint32_t* out_lens, uint16_t* tabs) {
    const uint32_t lane = threadIdx.x & 31, n_warps = (gridDim.x * blockDim.x) >> 5, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint16_t* table = tabs + (size_t)(warp % kSnappyWarps) * kSnappyMaxTable;
    for (uint32_t i = warp; i < n; i += n_warps) {
        const uint32_t c = warp_snappy_compress(bytes + offs[i], lens[i], out + out_offs[i], table, lane);
        if (lane == 0) out_lens[i] = c;
    }
}

extern "C" int b2_snappy_compress_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const uint32_t* offs, const uint32_t* lens,
                                        uint32_t n, void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens) {
    if (!c || !bytes || !offs || !lens || !out || !out_offs || !out_lens) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    if (nbytes > c->opt.max_batch_bytes || n > c->opt.max_msgs || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        if ((uint64_t)offs[i] + lens[i] > nbytes) { set_err("slice outside buffer"); return B2_E_INVAL; }
        if (!out_place(total, snappy_max_compressed_length(lens[i]), out_cap, &out_offs[i])) { set_err("output exceeds out_cap"); return B2_E_CAPACITY; }
    }
    CU(cudaSetDevice(c->opt.device));
    uint32_t* d_offs = c->d_frame_off; uint32_t* d_lens = c->d_slot; uint32_t* d_ooffs = c->d_frame_run; uint32_t* d_olens = (uint32_t*)c->d_aux;
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_offs, offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_lens, lens, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_ooffs, out_offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    if (n) k_snappy_compress_batch<<<c->n_sms * 4, 256, 0, c->stream>>>(c->d_bytes, d_offs, d_lens, n, c->d_unz, d_ooffs, d_olens, c->d_snappy_tab);
    CU(cudaMemcpyAsync(out_lens, d_olens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    if (total) CU(cudaMemcpyAsync(out, c->d_unz, total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}


// ---- leaf codecs with the REFERENCE's own signatures (seam 4: what a CompressHandler / ChecksumHandler body or any direct caller of
// butil::crc32c / butil::snappy would be re-pointed at).  They run on a process-wide default context (device $B2_DEVICE or 0, created on
// first use); one buffer per call is the latency-bound way to use a GPU — the batch forms above are the throughput path.
static std::mutex g_leaf_mu;
static b2_ctx* g_leaf_ctx = nullptr;
static b2_ctx* leaf_ctx(size_t need_bytes) {
    if (g_leaf_ctx && need_bytes + 4096 <= g_leaf_ctx->opt.max_batch_bytes) return g_leaf_ctx;
    if (g_leaf_ctx) { b2_ctx_destroy(g_leaf_ctx); g_leaf_ctx = nullptr; }
    b2_options o; memset(&o, 0, sizeof o);
    o.device = getenv("B2_DEVICE") ? atoi(getenv("B2_DEVICE")) : 0;
    size_t cap = 8u << 20; while (cap < need_bytes + 4096 && cap < (1ull << 30)) cap <<= 1;
    o.max_batch_bytes = (uint32_t)cap; o.max_msgs = 4096; o.max_runs = 16; o.max_resp_bytes = (uint32_t)(cap + cap / 4 + (1u << 20));
    if (b2_ctx_create(&o, &g_leaf_ctx) != B2_OK) g_leaf_ctx = nullptr;
    return g_leaf_ctx;
}
// butil::crc32c::Extend (src/butil/crc32c.h:24, crc32c.cc:379-454)
extern "C" uint32_t b2_crc32c_extend(uint32_t init_crc, const char* data, size_t n) {
    if (n == 0) return init_crc;
    std::lock_guard<std::mutex> g(g_leaf_mu);
    b2_ctx* c = leaf_ctx(n);
    if (!c || n > c->opt.max_batch_bytes) return 0;
    cudaSetDevice(c->opt.device);
    const uint32_t off = 0, len = (uint32_t)n; uint32_t out = 0;
    overwrites(c, kDevBatch);                       // (the private leaf context has no h2 batch or stream pass that could read its input)
    if (cudaMemcpyAsync(c->d_bytes, data, n, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return 0;
    cudaMemcpyAsync(c->d_frame_off, &off, 4, cudaMemcpyHostToDevice, c->stream);
    cudaMemcpyAsync(c->d_slot, &len, 4, cudaMemcpyHostToDevice, c->stream);
    k_crc32c_batch<<<1, 32, 0, c->stream>>>(c->d_bytes, c->d_frame_off, c->d_slot, 1, (uint32_t*)c->d_aux, c->d_crc_adv, init_crc);
    cudaMemcpyAsync(&out, c->d_aux, 4, cudaMemcpyDeviceToHost, c->stream);
    cudaStreamSynchronize(c->stream);
    return out;
}
// butil::snappy::MaxCompressedLength / RawCompress / GetUncompressedLength / RawUncompress (third_party/snappy/snappy.h:112-141)
extern "C" size_t b2_snappy_max_compressed_length(size_t n) { return 32 + n + n / 6; }
extern "C" void b2_snappy_raw_compress(const char* input, size_t input_length, char* compressed, size_t* compressed_length) {
    *compressed_length = 0;
    std::lock_guard<std::mutex> g(g_leaf_mu);
    b2_ctx* c = leaf_ctx(input_length + input_length / 4);
    if (!c) return;
    const uint32_t off = 0, len = (uint32_t)input_length; uint32_t ooff = 0, olen = 0;
    const uint8_t dummy = 0;
    if (b2_snappy_compress_batch(c, input_length ? (const void*)input : (const void*)&dummy, len, &off, &len, 1, compressed,
                                 (uint32_t)(((b2_snappy_max_compressed_length(input_length) + 15) & ~(size_t)15)), &ooff, &olen) == B2_OK) *compressed_length = olen;
}
extern "C" int b2_snappy_get_uncompressed_length(const char* compressed, size_t n, size_t* result) {   // varint32 preamble (snappy.cc:690-711)
    uint32_t v = 0, shift = 0; size_t k = 0;
    for (;;) {
        if (shift >= 32 || k >= n) return 0;
        const uint32_t b = (uint8_t)compressed[k++]; v |= (b & 0x7f) << shift;
        if (b < 128) break;
        shift += 7;
    }
    *result = v; return 1;
}
extern "C" int b2_snappy_raw_uncompress(const char* compressed, size_t compressed_length, char* uncompressed) {
    size_t ulen = 0;
    if (!b2_snappy_get_uncompressed_length(compressed, compressed_length, &ulen)) return 0;
    std::lock_guard<std::mutex> g(g_leaf_mu);
    b2_ctx* c = leaf_ctx(compressed_length > ulen ? compressed_length : ulen);
    if (!c) return 0;
    const uint32_t off = 0, len = (uint32_t)compressed_length; uint32_t ooff = 0; int32_t olen = -1;
    std::vector<char> tmp(((ulen + 15) & ~(size_t)15) + 16);
    if (b2_snappy_uncompress_batch(c, compressed, len, &off, &len, 1, tmp.data(), (uint32_t)tmp.size(), &ooff, &olen) != B2_OK || olen < 0 || (size_t)olen != ulen) return 0;
    memcpy(uncompressed, tmp.data() + ooff, ulen);
    return 1;
}

extern "C" int b2_hpack_reset(b2_ctx* c, uint32_t conn, uint32_t max_table_size) {
    if (!c || conn >= B2_HPACK_MAX_CONNS || max_table_size > 4096) { set_err("bad connection / table size"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    CU(cudaSetDevice(c->opt.device));
    k_hpack_reset<<<1, 1, 0, c->stream>>>(c->d_hpack, conn, max_table_size);
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// the items of a call on connection state, grouped by connection: the first item of every group, then n; false when a connection has two
template <class Conn> static bool conn_groups(uint32_t n, Conn conn, std::vector<uint32_t>& first) {
    for (uint32_t i = 0; i < n; i++) if (i == 0 || conn(i) != conn(i - 1)) first.push_back(i);
    first.push_back(n);
    for (size_t g = 0; g + 1 < first.size(); g++) for (size_t g2 = g + 1; g2 + 1 < first.size(); g2++) if (conn(first[g]) == conn(first[g2])) return false;
    return true;
}
extern "C" int b2_hpack_decode_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_hpack_block* blocks, uint32_t n,
                                     void* out, uint32_t per_block_cap, uint32_t* out_lens, int32_t* status, uint32_t* n_headers) {
    if (!c || !bytes || !blocks || !out || !out_lens || !status || !n_headers) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    if (nbytes > c->opt.max_batch_bytes || n > c->opt.max_msgs / 4 || (uint64_t)n * per_block_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    std::vector<uint32_t> conn(n), off(n), len(n), first;
    for (uint32_t i = 0; i < n; i++) {
        if (blocks[i].conn >= B2_HPACK_MAX_CONNS || (uint64_t)blocks[i].offset + blocks[i].length > nbytes) { set_err("bad block"); return B2_E_INVAL; }
        conn[i] = blocks[i].conn; off[i] = blocks[i].offset; len[i] = blocks[i].length;
    }
    if (!conn_groups(n, [&](uint32_t i) { return conn[i]; }, first)) { set_err("blocks of one connection must be adjacent"); return B2_E_INVAL; }
    const uint32_t n_groups = (uint32_t)first.size() - 1;
    CU(cudaSetDevice(c->opt.device));
    uint32_t* d_conn = c->d_frame_off; uint32_t* d_off = c->d_frame_run; uint32_t* d_len = c->d_slot;
    uint32_t* d_first = (uint32_t*)c->d_jobs; uint32_t* d_olens = (uint32_t*)c->d_aux; int32_t* d_st = (int32_t*)c->d_aux + n; uint32_t* d_nh = (uint32_t*)c->d_aux + 2 * (size_t)n;
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_conn, conn.data(), 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_off, off.data(), 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_len, len.data(), 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_first, first.data(), 4 * first.size(), cudaMemcpyHostToDevice, c->stream));
    if (n_groups) k_hpack_decode<<<(n_groups + 63) / 64, 64, 0, c->stream>>>(c->d_bytes, d_conn, d_off, d_len, d_first, n_groups, c->d_hpack, c->d_unz, per_block_cap, d_olens, d_st, d_nh);
    CU(cudaMemcpyAsync(out_lens, d_olens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(status, d_st, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(n_headers, d_nh, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    if (n) CU(cudaMemcpyAsync(out, c->d_unz, (size_t)n * per_block_cap, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

extern "C" int b2_h2_scan_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t max_frame_size,
                                b2_h2_frame* frames, uint32_t cap_per_run, uint32_t* n_frames, uint32_t* consumed, uint32_t* err) {
    if (!c || !bytes || !runs || !frames || !n_frames || !consumed || !err) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    if (nbytes > c->opt.max_batch_bytes || n_runs > c->opt.max_runs || (uint64_t)n_runs * cap_per_run * sizeof(b2_h2_frame) > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    for (uint32_t r = 0; r < n_runs; r++) if ((uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run outside buffer"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    static_assert(sizeof(b2_h2_frame) == sizeof(H2Frame), "frame layout");
    uint32_t* d_n = c->d_frame_off; uint32_t* d_cons = c->d_frame_run; uint32_t* d_err = c->d_slot;
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_meta, runs, sizeof(b2_run) * (size_t)n_runs, cudaMemcpyHostToDevice, c->stream));
    if (n_runs) k_h2_scan<<<(n_runs + 63) / 64, 64, 0, c->stream>>>(c->d_bytes, (const b2_run*)c->d_meta, n_runs, max_frame_size, (H2Frame*)c->d_unz, cap_per_run, d_n, d_cons, d_err);
    CU(cudaMemcpyAsync(n_frames, d_n, 4 * (size_t)n_runs, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(consumed, d_cons, 4 * (size_t)n_runs, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(err, d_err, 4 * (size_t)n_runs, cudaMemcpyDeviceToHost, c->stream));
    if (n_runs) CU(cudaMemcpyAsync(frames, c->d_unz, (size_t)n_runs * cap_per_run * sizeof(b2_h2_frame), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// ---- h2 connections: the state is allocated on first use (B2_H2_MAX_CONNS x ~128 KiB) ------------------------
static int h2_ensure(b2_ctx* c) {
    if (c->d_h2) return B2_OK;
    CU(cudaSetDevice(c->opt.device));
    const size_t n_streams = (size_t)c->h2_max_conns * c->h2_pending;
    CU(cudaMalloc(&c->d_h2, sizeof(H2Conn) * (size_t)c->h2_max_conns));
    if (cudaMalloc(&c->d_h2_streams, sizeof(H2Stream) * n_streams) != cudaSuccess || cudaMalloc(&c->d_h2_slots, n_streams * c->h2_stream_bytes) != cudaSuccess) {
        cudaFree(c->d_h2); cudaFree(c->d_h2_streams); c->d_h2 = nullptr; c->d_h2_streams = nullptr;
        set_err("h2 stream pool does not fit: lower b2_h2_configure's capacities"); return B2_E_NOMEM;
    }
    CU(cudaMemset(c->d_h2, 0, sizeof(H2Conn) * (size_t)c->h2_max_conns));
    CU(cudaMemset(c->d_h2_streams, 0xff, sizeof(H2Stream) * n_streams));           // id = -1: free
    return B2_OK;
}
// the second half of d_unz: input scratch of the h2 calls that must leave the first half alone, where the last h2 batch's out region
// stays for b2_h2_pack_responses' zero-copy sources (B2_H2_RESP_BODY_IN_OUT / _CT_IN_OUT)
static uint8_t* unz_upper(const b2_ctx* c) { return c->d_unz + c->opt.max_resp_bytes; }
static H2Pool h2_pool(const b2_ctx* c) { H2Pool p; p.streams = c->d_h2_streams; p.slots = c->d_h2_slots; p.pending = c->h2_pending; p.stream_bytes = c->h2_stream_bytes; return p; }
extern "C" int b2_h2_configure(b2_ctx* c, uint32_t max_conns, uint32_t max_pending, uint32_t stream_bytes) {
    if (!c || c->d_h2) { set_err("b2_h2_configure must precede the first h2 call on the context"); return B2_E_INVAL; }   // (b2_h2_ring_enable is an h2 call)
    if (max_conns == 0 || max_conns > B2_HPACK_MAX_CONNS || max_pending == 0 || max_pending > 65536 || stream_bytes < B2_H2_HEADER_BYTES + 16 || (stream_bytes & 15u)) {
        set_err("bad h2 capacities"); return B2_E_INVAL;
    }
    c->h2_max_conns = max_conns; c->h2_pending = max_pending; c->h2_stream_bytes = stream_bytes;
    return B2_OK;
}
extern "C" int b2_h2_conn_reset(b2_ctx* c, uint32_t conn) {
    if (!c || conn >= c->h2_max_conns) { set_err("bad connection index"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    k_h2_conn_reset<<<1, 1, 0, c->stream>>>(c->d_h2, c->d_hpack, conn, h2_pool(c));
    CU(cudaStreamSynchronize(c->stream));
    if (conn < c->h2_gunzip.size()) c->h2_gunzip[conn] = 0;        // (the kernel cleared the device bit with the rest of H2Conn)
    return B2_OK;
}
extern "C" int b2_h2_conn_set_gunzip(b2_ctx* c, uint32_t conn, int enable) {
    if (!c || conn >= c->h2_max_conns) { set_err("bad connection index"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    if (enable && !c->d_h2_gz_merge) {                            // once per context: the merge scratch of the select pass
        if (cudaMalloc(&c->d_h2_gz_merge, (size_t)c->opt.max_runs * B2_H2_HEADER_BYTES) != cudaSuccess) { c->d_h2_gz_merge = nullptr; set_err("cudaMalloc gunzip scratch failed"); return B2_E_NOMEM; }
    }
    if (c->h2_gunzip.size() < c->h2_max_conns) c->h2_gunzip.resize(c->h2_max_conns, 0);
    k_h2_set_gunzip<<<1, 1, 0, c->stream>>>(c->d_h2, conn, enable ? 1 : 0);
    CU(cudaStreamSynchronize(c->stream));
    c->h2_gunzip[conn] = enable ? 1 : 0;
    return B2_OK;
}
// the gunzip passes over a parsed batch (b2_h2_conn_set_gunzip), enqueued after the consume kernel and before the run statuses are fetched;
// nothing is launched unless a run is on an opted-in connection
static bool h2_gz_wanted(const b2_ctx* c, const b2_run* runs, uint32_t n_runs) {
    if (c->h2_gunzip.empty()) return false;
    for (uint32_t r = 0; r < n_runs; r++) if (c->h2_gunzip[runs[r].socket_id]) return true;
    return false;
}
template <class M>
static void h2_gz_launch(b2_ctx* c, uint32_t n_runs, b2_h2_run_status* d_rs, M* d_msgs, uint32_t per_run, uint32_t region) {
    uint32_t* d_gz = c->d_frame_off;                              // one word per descriptor slot (n_runs * per_run <= max_msgs)
    const uint32_t n_slots = n_runs * per_run;
    k_h2_gz_select<M><<<(n_runs + 31) / 32, 32, 0, c->stream>>>(c->d_bytes, (const b2_run*)c->d_meta, n_runs, c->d_h2, d_rs, d_msgs, per_run, c->d_unz, c->d_h2_gz_merge, d_gz);
    k_h2_gz_size<M><<<(n_slots + 63) / 64, 64, 0, c->stream>>>(c->d_bytes, n_runs, d_rs, d_msgs, per_run, c->d_unz, d_gz);
    k_h2_gz_place<M><<<(n_runs + 31) / 32, 32, 0, c->stream>>>(n_runs, d_rs, d_msgs, per_run, region, d_gz);
    k_h2_gz_inflate<M><<<(n_slots + 63) / 64, 64, 0, c->stream>>>(c->d_bytes, n_runs, d_rs, d_msgs, per_run, c->d_unz, d_gz);
}
// the answering passes of b2_h2_serve_batch (k_h2_serve .. k_h2_serve_gather), enqueued after the gunzip passes and before the run
// statuses are fetched.  Device scratch: per_run-strided records in the head rows and their reply offsets in d_frame_run, the list
// k_h2_pack reads in d_aux / d_slot, its lengths in d_frame_off (free once the gunzip passes ran), group_first in d_run_tile_base,
// the spans in d_refs, the packed replies in d_resp.
struct H2Serve { void* replies; uint32_t replies_cap; b2_h2_reply_span* spans; };
// the settings of the answering passes (b2_h2_serve_batch and k_h2_ring): the registered methods and the server identity
static H2ServeCfg h2_serve_cfg(const b2_ctx* c) {
    static_assert(sizeof(H2ServeCfg::identity) == sizeof(DevConfig::identity), "identity buffer");
    H2ServeCfg g; g.n_methods = c->cfg.n_methods; g.identity_len = c->cfg.identity_len; memcpy(g.identity, c->cfg.identity, sizeof g.identity); return g;
}
static void h2_serve_launch(b2_ctx* c, uint32_t n_runs, b2_h2_run_status* d_rs, b2_h2_msg* d_msgs, uint32_t per_run, uint32_t region, uint32_t reply_region) {
    static_assert(kHeadBytes >= sizeof(b2_h2_response) && sizeof(MsgAux) >= sizeof(b2_h2_response) && sizeof(uint4) == sizeof(b2_h2_reply_span), "serve scratch");
    b2_h2_response* d_strided = reinterpret_cast<b2_h2_response*>(c->d_heads);
    b2_h2_response* d_list = reinterpret_cast<b2_h2_response*>(c->d_aux);
    b2_h2_reply_span* d_spans = reinterpret_cast<b2_h2_reply_span*>(c->d_refs);
    uint32_t* d_first = c->d_run_tile_base;
    k_h2_serve<<<(n_runs + 31) / 32, 32, 0, c->stream>>>(c->d_bytes, (const b2_run*)c->d_meta, n_runs, c->d_methods, h2_serve_cfg(c), d_rs, d_msgs, per_run, c->d_unz, region,
                                                         d_strided, c->d_frame_run, reply_region, d_spans);
    k_h2_serve_scan<<<1, 32, 0, c->stream>>>(n_runs, d_spans, d_first);
    k_h2_serve_compact<<<(n_runs * per_run + 255) / 256, 256, 0, c->stream>>>(n_runs, per_run, d_spans, d_first, d_strided, c->d_frame_run, d_list, c->d_slot);
    k_h2_pack<<<(n_runs + kH2PackWarps - 1) / kH2PackWarps, kH2PackWarps * 32, 0, c->stream>>>(c->d_unz, c->d_bytes, c->d_unz, d_list, d_first, n_runs, c->d_h2,
                                                                                             c->d_resp, c->d_slot, c->d_frame_off);
    k_h2_serve_gather<<<(n_runs + kH2PackWarps - 1) / kH2PackWarps, kH2PackWarps * 32, 0, c->stream>>>(n_runs, d_first, c->d_slot, c->d_frame_off, c->d_resp, d_spans);
}
// the runs of an h2 batch or ring ticket: inside the buffer, one per connection, on a connection the context has
static bool h2_runs_ok(const b2_ctx* c, const b2_run* runs, uint32_t n_runs, uint32_t nbytes) {
    for (uint32_t r = 0; r < n_runs; r++) {
        if ((uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run outside buffer"); return false; }
        if (runs[r].socket_id >= c->h2_max_conns) { set_err("connection index out of range"); return false; }
        for (uint32_t q = 0; q < r; q++) if (runs[q].socket_id == runs[r].socket_id) { set_err("one run per connection and batch"); return false; }
    }
    return true;
}
// each run of an h2 batch or ring ticket owns `region` bytes of out (acks from its start, records / bodies from region / 4), per_run
// descriptors and reply_region bytes of the replies; fits: the least a run needs
struct H2Split { uint32_t region, per_run, reply_region; bool fits; };
static H2Split h2_split(uint32_t out_cap, uint32_t msg_cap, uint32_t replies_cap, uint32_t n_runs) {
    const uint32_t region = (out_cap / n_runs) & ~63u, per_run = msg_cap / n_runs;
    return { region, per_run, (replies_cap / n_runs) & ~63u, region >= 256 && per_run != 0 };
}
// ParseH2Message over a batch, server (b2_h2_msg) or client (b2_h2_call) connections: upload, the side's consume kernel (then the
// gunzip passes, and for b2_h2_serve_batch the answering passes), and a fetch of only what was produced.  The runs' parts of out and
// the descriptors (h2_split) come back in three strided copies, then the descriptors are compacted into one list (run order).
template <class M>
static int h2_parse_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                          b2_h2_run_status* rs, M* descs, uint32_t cap, uint32_t* n_descs, void* out, uint32_t out_cap, const H2Serve* serve = nullptr) {
    constexpr bool kClient = std::is_same<M, b2_h2_call>::value;
    if (!c || !bytes || !runs || !rs || !descs || !n_descs || !out || (serve && (!serve->replies || !serve->spans))) { set_err("null argument"); return B2_E_INVAL; }
    static_assert(sizeof(M) == 64 && sizeof(b2_h2_run_status) == 32, "h2 ABI layout");
    if (nbytes > c->opt.max_batch_bytes || n_runs > c->opt.max_runs || out_cap > 2ull * c->opt.max_resp_bytes || cap > c->opt.max_msgs ||
        (serve && serve->replies_cap > c->opt.max_resp_bytes)) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    *n_descs = 0;
    if (n_runs == 0) return B2_OK;
    if (!h2_runs_ok(c, runs, n_runs, nbytes)) return B2_E_INVAL;
    const auto [region, per_run, reply_region, fits] = h2_split(out_cap, cap, serve ? serve->replies_cap : 0, n_runs);
    if (!fits) { set_err(kClient ? "out_cap / call_cap too small for the number of runs" : "out_cap / msg_cap too small for the number of runs"); return B2_E_CAPACITY; }
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    b2_h2_run_status* d_rs = reinterpret_cast<b2_h2_run_status*>(c->d_run_status);      // 32 B each, like b2_run_status
    M* d_descs = reinterpret_cast<M*>(c->d_msgs);                                        // 64 B each, like b2_msg_desc
    overwrites(c, kDevInput | kDevBatch);
    CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_meta, runs, sizeof(b2_run) * (size_t)n_runs, cudaMemcpyHostToDevice, c->stream));
    if constexpr (kClient) k_h2_client_consume<<<(n_runs + 31) / 32, 32, 0, c->stream>>>(c->d_bytes, (const b2_run*)c->d_meta, n_runs, c->d_h2, c->d_hpack,
                                                                                          d_rs, d_descs, per_run, c->d_unz, region, h2_pool(c));
    else k_h2_consume<<<(n_runs + 31) / 32, 32, 0, c->stream>>>(c->d_bytes, (const b2_run*)c->d_meta, n_runs, c->d_h2, c->d_hpack, c->d_methods, c->cfg.n_methods,
                                                                 d_rs, d_descs, per_run, c->d_unz, region, h2_pool(c));
    if (h2_gz_wanted(c, runs, n_runs)) h2_gz_launch(c, n_runs, d_rs, d_descs, per_run, region);
    if constexpr (!kClient) {
        if (serve) {
            h2_serve_launch(c, n_runs, d_rs, d_descs, per_run, region, reply_region);
            CU(cudaMemcpyAsync(serve->spans, c->d_refs, sizeof(b2_h2_reply_span) * (size_t)n_runs, cudaMemcpyDeviceToHost, c->stream));
        }
    }
    CU(cudaMemcpyAsync(rs, d_rs, sizeof(b2_h2_run_status) * (size_t)n_runs, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    uint32_t total = 0, max_descs = 0, max_ctrl = 0, max_blob = 0, max_reply = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        total += rs[r].n_msgs; if (rs[r].n_msgs > max_descs) max_descs = rs[r].n_msgs;
        if (rs[r].ctrl_len > max_ctrl) max_ctrl = rs[r].ctrl_len;
        if (rs[r].first_msg > max_blob) max_blob = rs[r].first_msg;             // (the kernel reports the blob bytes it used here)
        if (serve && serve->spans[r].len > max_reply) max_reply = serve->spans[r].len;
    }
    if constexpr (!kClient) { if (total > cap) { set_err("msg_cap too small"); return B2_E_CAPACITY; } }
    std::vector<M> tmp((size_t)n_runs * (max_descs ? max_descs : 1));
    if (max_descs) CU(cudaMemcpy2DAsync(tmp.data(), sizeof(M) * (size_t)max_descs, d_descs, sizeof(M) * (size_t)per_run,
                                        sizeof(M) * (size_t)max_descs, n_runs, cudaMemcpyDeviceToHost, c->stream));
    if (max_ctrl) CU(cudaMemcpy2DAsync(out, region, c->d_unz, region, max_ctrl, n_runs, cudaMemcpyDeviceToHost, c->stream));
    if (max_blob) CU(cudaMemcpy2DAsync((uint8_t*)out + region / 4, region, c->d_unz + region / 4, region, max_blob, n_runs, cudaMemcpyDeviceToHost, c->stream));
    if (max_reply) CU(cudaMemcpy2DAsync(serve->replies, reply_region, c->d_resp, reply_region, max_reply, n_runs, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    total = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        if (rs[r].n_msgs) memcpy(descs + total, tmp.data() + (size_t)r * max_descs, sizeof(M) * (size_t)rs[r].n_msgs);
        rs[r].first_msg = total; total += rs[r].n_msgs;
    }
    // a server batch stays readable by b2_h2_pack_responses; a client batch leaves h2_last_in / h2_last_out at 0, so that it may not
    if constexpr (!kClient) { c->h2_last_in = nbytes; c->h2_last_out = (uint64_t)region * n_runs; }
    *n_descs = total;
    return B2_OK;
}
extern "C" int b2_h2_process_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                   b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t msg_cap, uint32_t* n_msgs,
                                   void* out, uint32_t out_cap) {
    return h2_parse_batch(c, bytes, nbytes, runs, n_runs, rs, msgs, msg_cap, n_msgs, out, out_cap);
}
extern "C" int b2_h2_serve_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                 b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t msg_cap, uint32_t* n_msgs, void* out, uint32_t out_cap,
                                 void* replies, uint32_t replies_cap, b2_h2_reply_span* spans) {
    static_assert(sizeof(b2_h2_reply_span) == 16, "reply span ABI layout");
    const H2Serve serve = { replies, replies_cap, spans };
    return h2_parse_batch(c, bytes, nbytes, runs, n_runs, rs, msgs, msg_cap, n_msgs, out, out_cap, &serve);
}

// the replies of b2_h2_pack_responses or of a turn (b2_h2_ring_turn_submit): the connection in range, every field inside its source
// (bytes, or the last batch's input / out for the zero-copy flags), content-type <= 256 and grpc-message <= 512 bytes, each reply's room
// in out placed at its bound (h2_reply_bound; total: the bytes placed), and replies of one connection adjacent (first: the connection groups)
static int h2_place_responses(const b2_ctx* c, uint32_t nbytes, const b2_h2_response* resps, uint32_t n, uint32_t out_cap,
                              uint32_t* out_offs, std::vector<uint32_t>& first, uint64_t& total) {
    for (uint32_t i = 0; i < n; i++) {
        const b2_h2_response& r = resps[i];
        const uint64_t body_lim = (r.flags & B2_H2_RESP_BODY_IN_INPUT) ? c->h2_last_in : (r.flags & B2_H2_RESP_BODY_IN_OUT) ? c->h2_last_out : nbytes;
        const uint64_t ct_lim = (r.flags & B2_H2_RESP_CT_IN_OUT) ? c->h2_last_out : nbytes;
        if (r.conn >= c->h2_max_conns || (uint64_t)r.body_off + r.body_len > body_lim || (uint64_t)r.content_type_off + r.content_type_len > ct_lim ||
            (uint64_t)r.grpc_message_off + r.grpc_message_len > nbytes || r.content_type_len > 256 || r.grpc_message_len > 512) { set_err("bad response descriptor"); return B2_E_INVAL; }
        if ((r.flags & (B2_H2_RESP_BODY_IN_OUT | B2_H2_RESP_CT_IN_OUT)) && c->h2_last_out > c->opt.max_resp_bytes) { set_err("last h2 out buffer too large to stay resident"); return B2_E_CAPACITY; }
        const uint64_t need = h2_reply_bound(r.body_len, r.content_type_len, r.grpc_message_len);
        if (!out_place(total, need, out_cap, &out_offs[i])) { set_err("out_cap too small"); return B2_E_CAPACITY; }
    }
    if (!conn_groups(n, [&](uint32_t i) { return resps[i].conn; }, first)) { set_err("responses of one connection must be adjacent"); return B2_E_INVAL; }
    return B2_OK;
}
extern "C" int b2_h2_pack_responses(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_h2_response* resps, uint32_t n,
                                    void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens) {
    if (!c || (!bytes && nbytes) || !resps || !out || !out_offs || !out_lens) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    static_assert(sizeof(b2_h2_response) == 48, "h2 response ABI layout");
    if (nbytes > c->opt.max_resp_bytes || n > c->opt.max_msgs || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (n == 0) return B2_OK;
    std::vector<uint32_t> first;
    uint64_t total = 0;
    { int rc = h2_place_responses(c, nbytes, resps, n, out_cap, out_offs, first, total); if (rc != B2_OK) return rc; }
    const uint32_t n_groups = (uint32_t)first.size() - 1;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    b2_h2_response* d_resps = reinterpret_cast<b2_h2_response*>(c->d_msgs);       // 48 B <= 64 B per entry
    uint32_t* d_first = c->d_frame_off; uint32_t* d_offs = c->d_frame_run; uint32_t* d_lens = c->d_slot;
    uint8_t* d_aux = unz_upper(c);
    overwrites(c, kDevBatch);
    if (nbytes) CU(cudaMemcpyAsync(d_aux, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_resps, resps, sizeof(b2_h2_response) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_first, first.data(), 4 * first.size(), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_offs, out_offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    k_h2_pack<<<(n_groups + kH2PackWarps - 1) / kH2PackWarps, kH2PackWarps * 32, 0, c->stream>>>(d_aux, c->d_bytes, c->d_unz, d_resps, d_first, n_groups, c->d_h2, c->d_resp, d_offs, d_lens);
    CU(cudaMemcpyAsync(out_lens, d_lens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(out, c->d_resp, (size_t)total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// the requests of b2_h2_pack_requests or of a client ring ticket: every descriptor inside bytes, header blocks that fit the kernel's
// fragment (kH2ReqFragCap), requests of one connection adjacent (first: the connection groups), and each request's room in out placed
// (results[i].out_off, the rest of results[i] zeroed; total: the bytes placed)
static int h2_place_requests(const b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_h2_request* reqs, uint32_t n, uint32_t out_cap,
                             b2_h2_request_result* results, std::vector<uint32_t>& first, uint64_t& total) {
    for (uint32_t i = 0; i < n; i++) {
        const b2_h2_request& r = reqs[i];
        if (r.conn >= c->h2_max_conns || (uint64_t)r.path_off + r.path_len > nbytes || (uint64_t)r.authority_off + r.authority_len > nbytes ||
            (uint64_t)r.content_type_off + r.content_type_len > nbytes || (uint64_t)r.body_off + r.body_len > nbytes ||
            (uint64_t)r.extra_off + r.extra_len > nbytes) { set_err("bad request descriptor"); return B2_E_INVAL; }
        // the encoded header block must fit the kernel's shared-memory fragment: every header costs at most its bytes + 2 x 3 length bytes + 1
        uint64_t hdr = 4 * 16 + 64 + (uint64_t)r.path_len + r.authority_len + r.content_type_len + 16 + 32, n_extra = 0;
        for (uint32_t at = 0; at + 4 <= r.extra_len;) {
            const uint8_t* e = static_cast<const uint8_t*>(bytes) + r.extra_off + at;
            const uint32_t nl = e[0] | ((uint32_t)e[1] << 8), vl = e[2] | ((uint32_t)e[3] << 8);
            if (at + 4 + nl + vl > r.extra_len) { set_err("truncated extra header record"); return B2_E_INVAL; }
            if (nl + vl > kH2ReqFragCap / 2) { set_err("header too long"); return B2_E_INVAL; }
            hdr += nl + vl + 8; n_extra++; at += 4 + nl + vl;
        }
        if (hdr > kH2ReqFragCap || r.path_len + 16 > kH2ReqFragCap / 2 || r.authority_len + 16 > kH2ReqFragCap / 2 || r.content_type_len + 16 > kH2ReqFragCap / 2) { set_err("header block too long"); return B2_E_INVAL; }
        const uint64_t data = (uint64_t)r.body_len + 5;
        const uint64_t need = 58 + hdr + 9 + data + 9 * (data / 16384 + 4) + 13 + 16;
        results[i].status = 0; results[i].stream_id = 0; results[i].out_len = 0;
        if (!out_place(total, need, out_cap, &results[i].out_off)) { set_err("out_cap too small"); return B2_E_CAPACITY; }
    }
    if (!conn_groups(n, [&](uint32_t i) { return reqs[i].conn; }, first)) { set_err("requests of one connection must be adjacent"); return B2_E_INVAL; }
    return B2_OK;
}
// client side of h2: see include/b2rpc.h
extern "C" int b2_h2_pack_requests(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_h2_request* reqs, uint32_t n,
                                   void* out, uint32_t out_cap, b2_h2_request_result* results) {
    if (!c || !bytes || !reqs || !out || !results) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    static_assert(sizeof(b2_h2_request) == 48 && sizeof(b2_h2_request_result) == 16, "h2 request ABI layout");
    if (nbytes > c->opt.max_resp_bytes || n > c->opt.max_msgs || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (n == 0) return B2_OK;
    std::vector<uint32_t> first;
    uint64_t total = 0;
    { int rc = h2_place_requests(c, bytes, nbytes, reqs, n, out_cap, results, first, total); if (rc != B2_OK) return rc; }
    const uint32_t n_groups = (uint32_t)first.size() - 1;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    b2_h2_request* d_reqs = reinterpret_cast<b2_h2_request*>(c->d_msgs);          // 48 B <= 64 B per entry
    b2_h2_request_result* d_res = reinterpret_cast<b2_h2_request_result*>(c->d_aux);
    static_assert(sizeof(MsgAux) >= sizeof(b2_h2_request_result), "results live in the aux array");
    uint32_t* d_first = c->d_frame_off;
    uint8_t* d_in = unz_upper(c);
    overwrites(c, kDevBatch);
    CU(cudaMemcpyAsync(d_in, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_reqs, reqs, sizeof(b2_h2_request) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_res, results, sizeof(b2_h2_request_result) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_first, first.data(), 4 * first.size(), cudaMemcpyHostToDevice, c->stream));
    k_h2_pack_req<<<(n_groups + kH2PackWarps - 1) / kH2PackWarps, kH2PackWarps * 32, 0, c->stream>>>(d_in, d_reqs, d_first, n_groups, c->d_h2, c->d_resp, d_res, h2_pool(c));
    CU(cudaMemcpyAsync(results, d_res, sizeof(b2_h2_request_result) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(out, c->d_resp, (size_t)total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}
extern "C" int b2_h2_conn_peer_update(b2_ctx* c, uint32_t conn, const b2_h2_peer_update* u) {
    if (!c || !u) { set_err("null argument"); return B2_E_INVAL; }
    static_assert(sizeof(b2_h2_peer_update) == 24, "peer update ABI layout");
    if ((u->set & B2_H2_PEER_MAX_FRAME_SIZE) && (u->max_frame_size < 16384u || u->max_frame_size > 16777215u)) { set_err("max_frame_size out of range"); return B2_E_INVAL; }   // ParseH2Settings :166-211
    if ((u->set & B2_H2_PEER_STREAM_WINDOW) && u->stream_window_size > 0x7fffffffu) { set_err("stream_window_size out of range"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    if (conn >= c->h2_max_conns) { set_err("conn out of range"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    int* d_rc = reinterpret_cast<int*>(c->d_slot); int h_rc = 0;
    k_h2_peer_update<<<1, 1, 0, c->stream>>>(c->d_h2, conn, *u, d_rc);
    CU(cudaMemcpyAsync(&h_rc, d_rc, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (h_rc != 0) { set_err("connection window would pass 2^31 - 1 (FLOW_CONTROL_ERROR)"); return B2_E_INVAL; }
    return B2_OK;
}
extern "C" int b2_h2_conn_set_next_stream_id(b2_ctx* c, uint32_t conn, uint32_t next_id) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    if (conn >= c->h2_max_conns) { set_err("conn out of range"); return B2_E_INVAL; }
    CU(cudaSetDevice(c->opt.device));
    k_h2_set_next_stream_id<<<1, 1, 0, c->stream>>>(c->d_h2, conn, next_id);
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// the receiving half of a client connection: see include/b2rpc.h
extern "C" int b2_h2_client_conn_reset(b2_ctx* c, uint32_t conn) {
    if (!c || conn >= c->h2_max_conns) { set_err("bad connection index"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    k_h2_client_conn_reset<<<1, 1, 0, c->stream>>>(c->d_h2, c->d_hpack, conn, h2_pool(c));
    CU(cudaStreamSynchronize(c->stream));
    if (conn < c->h2_gunzip.size()) c->h2_gunzip[conn] = 0;
    return B2_OK;
}
extern "C" int b2_h2_client_abandon_streams(b2_ctx* c, uint32_t conn, const uint32_t* stream_ids, uint32_t n) {
    if (!c || (!stream_ids && n)) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, true)) return B2_E_INVAL;
    if (conn >= c->h2_max_conns) { set_err("bad connection index"); return B2_E_INVAL; }
    if ((uint64_t)n * 4 > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }   // (the ids go to unz_upper)
    if (n == 0) return B2_OK;
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    uint32_t* d_ids = reinterpret_cast<uint32_t*>(unz_upper(c));
    CU(cudaMemcpyAsync(d_ids, stream_ids, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    k_h2_client_abandon<<<1, 1, 0, c->stream>>>(c->d_h2, conn, d_ids, n, h2_pool(c));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}
extern "C" int b2_h2_client_process_batch(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                          b2_h2_run_status* rs, b2_h2_call* calls, uint32_t call_cap, uint32_t* n_calls,
                                          void* out, uint32_t out_cap) {
    return h2_parse_batch(c, bytes, nbytes, runs, n_runs, rs, calls, call_cap, n_calls, out, out_cap);
}

// the frame of every request, placed with out_place at its worst-case size (b2_pack_requests, b2_client_ring_submit); total: the bytes placed
static int place_requests(uint32_t nbytes, const b2_request* reqs, uint32_t n, uint32_t out_cap, uint32_t* out_offs, uint64_t& total) {
    for (uint32_t i = 0; i < n; i++) {
        const b2_request& r = reqs[i];
        if ((uint64_t)r.payload_off + r.payload_len > nbytes || (uint64_t)r.attachment_off + r.attachment_len > nbytes) { set_err("payload outside buffer"); return B2_E_INVAL; }
        const uint64_t pb = 6ull + r.payload_len;
        const uint64_t need = 12 + 512 + (r.compress_type == B2_COMPRESS_TYPE_SNAPPY ? snappy_max_compressed_length((uint32_t)pb) : pb) + r.attachment_len;
        if (!out_place(total, need, out_cap, &out_offs[i])) { set_err("out_cap too small"); return B2_E_CAPACITY; }
    }
    return B2_OK;
}
extern "C" int b2_pack_requests(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_request* reqs, uint32_t n,
                                void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens) {
    if (!c || (!bytes && nbytes) || !reqs || !out || !out_offs || !out_lens) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    static_assert(sizeof(b2_request) == 64 && sizeof(ReqDesc) == 64, "request ABI layout");
    if (nbytes > c->opt.max_batch_bytes || n > c->opt.max_msgs || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (n == 0) return B2_OK;
    uint64_t total = 0;
    const int rc = place_requests(nbytes, reqs, n, out_cap, out_offs, total);
    if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    ReqDesc* d_reqs = reinterpret_cast<ReqDesc*>(c->d_msgs);
    uint32_t* d_offs = c->d_frame_off; uint32_t* d_lens = c->d_slot;
    overwrites(c, kDevInput | kDevBatch);
    if (nbytes) CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_reqs, reqs, sizeof(b2_request) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_offs, out_offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    k_pack_requests<<<c->n_sms * 4, 256, 0, c->stream>>>(c->d_bytes, d_reqs, n, c->d_methods, c->cfg.n_methods, c->d_resp, d_offs, d_lens, c->d_unz, c->d_snappy_tab, c->d_crc_adv);
    CU(cudaMemcpyAsync(out_lens, d_lens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(out, c->d_resp, (size_t)total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// the frame of every reply, placed with out_place at its worst-case size (b2_pack_responses, b2_ring_turn_submit); total: the bytes placed
static int place_replies(const void* bytes, uint32_t nbytes, const b2_reply* reps, uint32_t n, uint32_t out_cap, uint32_t* out_offs, uint64_t& total) {
    for (uint32_t i = 0; i < n; i++) {
        const b2_reply& r = reps[i];
        if ((uint64_t)r.body_off + r.body_len > nbytes || (uint64_t)r.attachment_off + r.attachment_len > nbytes || (uint64_t)r.error_text_off + r.error_text_len > nbytes ||
            (uint64_t)r.checksum_value_off + r.checksum_value_len > nbytes || (r.extra_streams_off & 7u) || (uint64_t)r.extra_streams_off + 8ull * r.n_extra_streams > nbytes ||
            r.user_fields_off > nbytes) { set_err("reply field outside buffer"); return B2_E_INVAL; }
        uint64_t uf = 0, at = r.user_fields_off;                       // every record must lie inside the buffer: the kernel walks them
        for (uint32_t k = 0; k < r.n_user_fields; k++) {
            if (at + 8 > nbytes) { set_err("user field outside buffer"); return B2_E_INVAL; }
            uint32_t kl, vl; memcpy(&kl, static_cast<const uint8_t*>(bytes) + at, 4); memcpy(&vl, static_cast<const uint8_t*>(bytes) + at + 4, 4);
            if (at + 8 + (uint64_t)kl + vl > nbytes) { set_err("user field outside buffer"); return B2_E_INVAL; }
            uf += 24ull + kl + vl; at += 8ull + kl + vl;
        }
        const uint64_t body = r.compress_type == B2_COMPRESS_TYPE_SNAPPY ? snappy_max_compressed_length(r.body_len) : r.body_len;
        const uint64_t need = 12 + 128 + r.error_text_len + r.checksum_value_len + 11ull * r.n_extra_streams + uf + body + r.attachment_len;
        if (!out_place(total, need, out_cap, &out_offs[i])) { set_err("out_cap too small"); return B2_E_CAPACITY; }
    }
    return B2_OK;
}
// SendRpcResponse for replies the host produced: see include/b2rpc.h
extern "C" int b2_pack_responses(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_reply* reps, uint32_t n,
                                 void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens) {
    if (!c || (!bytes && nbytes) || !reps || !out || !out_offs || !out_lens) { set_err("null argument"); return B2_E_INVAL; }
    if (ring_refuses(c, false)) return B2_E_INVAL;
    static_assert(sizeof(b2_reply) == 88 && sizeof(ReplyDesc) == 88, "reply ABI layout");
    if (nbytes > c->opt.max_batch_bytes || (uint64_t)n * sizeof(b2_reply) > (uint64_t)c->opt.max_msgs * 64 || out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (n == 0) return B2_OK;
    uint64_t total = 0;
    const int rc = place_replies(bytes, nbytes, reps, n, out_cap, out_offs, total);
    if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    ReplyDesc* d_reps = reinterpret_cast<ReplyDesc*>(c->d_msgs);
    uint32_t* d_offs = c->d_frame_off; uint32_t* d_lens = c->d_slot;
    overwrites(c, kDevInput | kDevBatch);
    if (nbytes) CU(cudaMemcpyAsync(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_reps, reps, sizeof(b2_reply) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_offs, out_offs, 4 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    k_pack_responses<<<c->n_sms * 4, 256, 0, c->stream>>>(c->d_bytes, d_reps, n, c->d_resp, d_offs, d_lens, c->d_unz, c->d_snappy_tab, c->d_crc_adv);
    CU(cudaMemcpyAsync(out_lens, d_lens, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(out, c->d_resp, (size_t)total, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return B2_OK;
}

// ---- h2/gRPC on the latency path: k_h2_ring on the same submit ring (include/b2rpc.h, b2_h2_ring_enable) ---------------------------
// the kernel arguments at each (re)launch: the slot parts of b2_h2_ring_enable, and the methods and identity as they are now
static H2RingDev h2_ring_dev(const b2_ctx* c) {
    H2RingDev H = c->h2r_dev;
    H.conns = c->d_h2; H.hps = c->d_hpack; H.methods = c->d_methods; H.n_methods = c->cfg.n_methods; H.pool = h2_pool(c);
    H.cfg = h2_serve_cfg(c);
    // the scratch of b2_h2_serve_batch (h2_parse_batch, h2_gz_launch, h2_serve_launch)
    H.rs = reinterpret_cast<b2_h2_run_status*>(c->d_run_status); H.msgs = reinterpret_cast<b2_h2_msg*>(c->d_msgs); H.out = c->d_unz;
    H.merge = c->d_h2_gz_merge; H.gz = c->d_frame_off;
    H.strided = reinterpret_cast<b2_h2_response*>(c->d_heads); H.strided_offs = c->d_frame_run;
    H.list = reinterpret_cast<b2_h2_response*>(c->d_aux); H.list_offs = c->d_slot; H.first = c->d_run_tile_base;
    H.spans = reinterpret_cast<b2_h2_reply_span*>(c->d_refs); H.replies = c->d_resp;
    return H;
}
// b2_h2_ring_enable, and b2_h2_ring_turn_enable with max_resps > 0: the host-reply parts of the slot and their device scratch too
static int h2_ring_setup(b2_ctx* c, const char* call, uint32_t max_bytes, uint32_t msg_cap, uint32_t out_cap, uint32_t replies_cap,
                         uint32_t max_resps, uint32_t resp_out_cap) {
    if (c->ring_kind != RingKind::none) { set_err("%s: once, before the context's first ring call, and not with another ring kind", call); return B2_E_INVAL; }
    if (max_bytes == 0 || msg_cap == 0 || out_cap == 0 || replies_cap == 0) { set_err("capacities must be non-zero"); return B2_E_INVAL; }
    if (max_bytes > c->opt.max_batch_bytes || out_cap > 2ull * c->opt.max_resp_bytes || msg_cap > c->opt.max_msgs || replies_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    static_assert(sizeof(RingSlotHdr) + sizeof(H2RingArgs) <= 256, "h2 ring slot header");
    // [RingSlotHdr | args | runs | staged input | (host-reply block) | statuses | msgs | spans | out | replies | (reply lengths | frames)]
    const uint64_t runs = (uint64_t)c->opt.max_runs;
    SlotLayout L;
    H2RingDev& H = c->h2r_dev;
    H.off_args = sizeof(RingSlotHdr);
    c->ring_dev.off_runs = L.add(runs * sizeof(b2_run));
    c->ring_dev.off_in = L.add((uint64_t)max_bytes + 16);
    H2TurnDev& Q = c->h2t_dev;
    if (max_resps) Q.off_resps = L.add(h2r_turn_block(max_resps, max_resps));
    H.off_rs = L.add(runs * sizeof(b2_h2_run_status));
    H.off_msgs = L.add((uint64_t)msg_cap * sizeof(b2_h2_msg));
    H.off_spans = L.add(runs * sizeof(b2_h2_reply_span));
    H.off_out = L.add((uint64_t)out_cap + 16);
    H.off_replies = L.add((uint64_t)replies_cap + 16);
    if (max_resps) {
        Q.off_resp_lens = L.add(max_resps * 4ull);
        Q.off_resp_out = L.add((uint64_t)resp_out_cap + 16);
        // the device scratch: [block | lengths | frames]
        const uint64_t block = h2r_turn_block(max_resps, max_resps), lens = (max_resps * 4ull + 15u) & ~15ull;
        if (cudaMalloc((void**)&Q.turn, block + lens + resp_out_cap + 16) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the turn's reply scratch failed"); return B2_E_NOMEM; }
        Q.turn_lens = reinterpret_cast<uint32_t*>(Q.turn + block); Q.turn_out = Q.turn + block + lens;
    }
    rc = ring_alloc(c, L.end); if (rc != B2_OK) return rc;
    if (max_resps) CU(cudaFuncSetAttribute(k_h2_ring<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kH2RingSmem));
    else CU(cudaFuncSetAttribute(k_h2_ring<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kH2RingSmem));
    c->h2r_max_bytes = max_bytes; c->h2r_msg_cap = msg_cap; c->h2r_out_cap = out_cap; c->h2r_replies_cap = replies_cap;
    c->h2r_max_resps = max_resps; c->h2r_resp_out_cap = resp_out_cap;
    c->ring_kind = RingKind::h2_server;
    return B2_OK;
}
extern "C" int b2_h2_ring_enable(b2_ctx* c, uint32_t max_bytes, uint32_t msg_cap, uint32_t out_cap, uint32_t replies_cap) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    return h2_ring_setup(c, "b2_h2_ring_enable", max_bytes, msg_cap, out_cap, replies_cap, 0, 0);
}
extern "C" int b2_h2_ring_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t* ticket) {
    if (!c || !bytes || !runs || !ticket || n_runs == 0) { set_err("null argument"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::h2_server) { set_err("b2_h2_ring_enable first"); return B2_E_INVAL; }
    // the argument checks of b2_h2_serve_batch (h2_parse_batch) with the caps of b2_h2_ring_enable, and the slot's staging size
    if (nbytes > c->h2r_max_bytes) { set_err("batch larger than b2_h2_ring_enable's max_bytes: use b2_h2_serve_batch"); return B2_E_CAPACITY; }
    if (n_runs > c->opt.max_runs) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    if (!h2_runs_ok(c, runs, n_runs, nbytes)) return B2_E_INVAL;
    const H2Split sp = h2_split(c->h2r_out_cap, c->h2r_msg_cap, c->h2r_replies_cap, n_runs);
    if (!sp.fits) { set_err("out_cap / msg_cap too small for the number of runs"); return B2_E_CAPACITY; }
    const H2RingArgs a = { sp.per_run, sp.region, sp.reply_region, h2_gz_wanted(c, runs, n_runs) ? 1u : 0u, 0, 0, { 0, 0 } };
    uint8_t* slot = ring_claim(c, "b2_h2_ring_wait");
    if (!slot) return B2_E_CAPACITY;
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    memcpy(slot + c->h2r_dev.off_args, &a, sizeof a);
    return ring_ring(c, h, bytes, ticket);
}
// the served half of a collected k_h2_ring ticket
static void h2_ring_result(b2_ctx* c, uint32_t ticket, const uint8_t* slot, b2_h2_ring_result* out) {
    const RingSlotHdr* h = reinterpret_cast<const RingSlotHdr*>(slot);
    const H2RingDev& L = c->h2r_dev;
    const H2RingArgs* a = reinterpret_cast<const H2RingArgs*>(slot + L.off_args);
    const uint32_t n_runs = h->n_runs;
    const b2_h2_run_status* rs = reinterpret_cast<const b2_h2_run_status*>(slot + L.off_rs);
    uint32_t n_msgs = 0;
    for (uint32_t r = 0; r < n_runs; r++) n_msgs += rs[r].n_msgs;
    memset(out, 0, sizeof *out);
    out->runs = rs; out->n_runs = n_runs; out->n_msgs = n_msgs;
    out->msgs = reinterpret_cast<const b2_h2_msg*>(slot + L.off_msgs);
    out->out = slot + L.off_out; out->region = a->region;     // (h2_split's, as the submission placed it; 0 on a turn without runs)
    out->replies = slot + L.off_replies; out->spans = reinterpret_cast<const b2_h2_reply_span*>(slot + L.off_spans);
    if (n_msgs > c->h2r_msg_cap) { out->n_msgs = 0; out->status = B2_E_CAPACITY; }
    // the most recent ticket's input and out regions stay on the device: b2_h2_pack_responses may take bodies and content-types from them
    if (ticket + 1 == c->ring_next) { c->h2_last_in = h->nbytes; c->h2_last_out = (uint64_t)out->region * n_runs; }
}
extern "C" int b2_h2_ring_wait(b2_ctx* c, uint32_t ticket, b2_h2_ring_result* out) {
    static_assert(sizeof(b2_h2_ring_result) == 64, "h2 ring result ABI layout");
    int rc;
    const uint8_t* slot = ring_collect(c, c && out && c->ring_kind == RingKind::h2_server, ticket, "bad h2 ring ticket", rc);
    if (!slot) return rc;
    h2_ring_result(c, ticket, slot, out);
    return B2_OK;
}

// ---- a gRPC server's turn on the latency path: k_h2_ring with the host-reply phase (include/b2rpc.h, b2_h2_ring_turn_enable) ----------
extern "C" int b2_h2_ring_turn_enable(b2_ctx* c, uint32_t max_bytes, uint32_t msg_cap, uint32_t out_cap, uint32_t replies_cap,
                                      uint32_t max_resps, uint32_t resp_out_cap) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    if (max_resps == 0 || resp_out_cap == 0) { set_err("capacities must be non-zero"); return B2_E_INVAL; }
    // the limits of b2_h2_pack_responses, which reads the ticket's bytes
    if (max_bytes > c->opt.max_resp_bytes || max_resps > c->opt.max_msgs || resp_out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    return h2_ring_setup(c, "b2_h2_ring_turn_enable", max_bytes, msg_cap, out_cap, replies_cap, max_resps, resp_out_cap);
}
extern "C" int b2_h2_ring_turn_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                      const b2_h2_response* resps, uint32_t n_resps, uint32_t* ticket) {
    if (!c || !bytes || !ticket || (!runs && n_runs) || (!resps && n_resps)) { set_err("null argument"); return B2_E_INVAL; }
    if (n_runs == 0 && n_resps == 0) { set_err("a turn carries runs, host replies or both"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::h2_server || !c->h2r_max_resps) { set_err("b2_h2_ring_turn_enable first"); return B2_E_INVAL; }
    // the checks of b2_h2_ring_submit for the runs, then those of b2_h2_pack_responses for the replies, with the enable-time caps
    if (nbytes > c->h2r_max_bytes) { set_err("turn larger than b2_h2_ring_turn_enable's max_bytes: use the batch calls"); return B2_E_CAPACITY; }
    if (n_runs > c->opt.max_runs || n_resps > c->h2r_max_resps) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    H2Split sp = { 0, 0, 0, true };
    if (n_runs) {
        if (!h2_runs_ok(c, runs, n_runs, nbytes)) return B2_E_INVAL;
        sp = h2_split(c->h2r_out_cap, c->h2r_msg_cap, c->h2r_replies_cap, n_runs);
        if (!sp.fits) { set_err("out_cap / msg_cap too small for the number of runs"); return B2_E_CAPACITY; }
    }
    // the zero-copy sources are the previous ticket's device buffers, which this ticket's pull overwrites
    for (uint32_t i = 0; i < n_resps; i++)
        if (resps[i].flags & (B2_H2_RESP_BODY_IN_INPUT | B2_H2_RESP_BODY_IN_OUT | B2_H2_RESP_CT_IN_OUT)) { set_err("a turn's replies index its own bytes: no zero-copy flags"); return B2_E_INVAL; }
    std::vector<uint32_t> first, offs(n_resps);
    uint64_t total = 0;
    if (n_resps) { int rc = h2_place_responses(c, nbytes, resps, n_resps, c->h2r_resp_out_cap, offs.data(), first, total); if (rc != B2_OK) return rc; }
    uint8_t* slot = ring_claim(c, "b2_h2_ring_turn_wait");
    if (!slot) return B2_E_CAPACITY;
    const uint32_t n_groups = n_resps ? (uint32_t)first.size() - 1 : 0u;
    const H2RingArgs a = { sp.per_run, sp.region, sp.reply_region, n_runs && h2_gz_wanted(c, runs, n_runs) ? 1u : 0u, n_resps, n_groups, { 0, 0 } };
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    uint8_t* block = slot + c->h2t_dev.off_resps;                 // the host-reply block the kernel pulls: records, placed offsets, group_first
    if (n_resps) {
        memcpy(block, resps, sizeof(b2_h2_response) * (size_t)n_resps);
        memcpy(block + h2r_turn_offs_off(n_resps), offs.data(), 4 * (size_t)n_resps);
        memcpy(block + h2r_turn_first_off(n_resps), first.data(), 4 * first.size());
    }
    memcpy(slot + c->h2r_dev.off_args, &a, sizeof a);
    return ring_ring(c, h, bytes, ticket);
}
extern "C" int b2_h2_ring_turn_wait(b2_ctx* c, uint32_t ticket, b2_h2_ring_turn_result* out) {
    static_assert(sizeof(b2_h2_ring_turn_result) == 96, "h2 ring turn result ABI layout");
    int rc;
    const uint8_t* slot = ring_collect(c, c && out && c->ring_kind == RingKind::h2_server && c->h2r_max_resps, ticket, "bad h2 ring turn ticket", rc);
    if (!slot) return rc;
    memset(out, 0, sizeof *out);
    h2_ring_result(c, ticket, slot, &out->ring);
    const H2TurnDev& Q = c->h2t_dev;
    out->n_resps = reinterpret_cast<const H2RingArgs*>(slot + c->h2r_dev.off_args)->n_resps;
    out->resp_offs = reinterpret_cast<const uint32_t*>(slot + Q.off_resps + h2r_turn_offs_off(out->n_resps));
    out->resp_lens = reinterpret_cast<const uint32_t*>(slot + Q.off_resp_lens);
    out->resp_out = slot + Q.off_resp_out;
    return B2_OK;
}

// ---- h2/gRPC client connections on the latency path: k_h2_client_ring on the same submit ring (include/b2rpc.h, b2_h2_client_ring_enable)
static H2ClientRingDev h2_client_ring_dev(const b2_ctx* c) {
    H2ClientRingDev H = c->h2c_dev;
    H.conns = c->d_h2; H.hps = c->d_hpack; H.pool = h2_pool(c);
    // the scratch of b2_h2_client_process_batch (h2_parse_batch, h2_gz_launch); the request block in the head rows, which the client parse
    // leaves alone (b2_h2_pack_requests' own d_msgs / d_aux / d_frame_off would overlap the calls and gz words), the frames in d_resp
    static_assert(kHeadBytes >= sizeof(b2_h2_request) + sizeof(b2_h2_request_result) + 4, "request block in the head rows");
    H.rs = reinterpret_cast<b2_h2_run_status*>(c->d_run_status); H.calls = reinterpret_cast<b2_h2_call*>(c->d_msgs); H.out = c->d_unz;
    H.merge = c->d_h2_gz_merge; H.gz = c->d_frame_off; H.first = c->d_run_tile_base;
    H.reqs = c->d_heads; H.req_out = c->d_resp;
    return H;
}
extern "C" int b2_h2_client_ring_enable(b2_ctx* c, uint32_t max_bytes, uint32_t call_cap, uint32_t out_cap, uint32_t max_reqs, uint32_t req_out_cap) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::none) { set_err("b2_h2_client_ring_enable: once, before the context's first ring call, and not with another ring kind"); return B2_E_INVAL; }
    if (max_bytes == 0 || call_cap == 0 || out_cap == 0 || max_reqs == 0 || req_out_cap == 0) { set_err("capacities must be non-zero"); return B2_E_INVAL; }
    // the limits of b2_h2_client_process_batch and b2_h2_pack_requests, both of which read the ticket's bytes
    if (max_bytes > c->opt.max_batch_bytes || max_bytes > c->opt.max_resp_bytes || call_cap > c->opt.max_msgs || out_cap > 2ull * c->opt.max_resp_bytes ||
        max_reqs > c->opt.max_msgs || req_out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    int rc = h2_ensure(c); if (rc != B2_OK) return rc;
    CU(cudaSetDevice(c->opt.device));
    static_assert(sizeof(RingSlotHdr) + sizeof(H2ClientRingArgs) <= 256, "h2 client ring slot header");
    // [RingSlotHdr | args | runs | staged input | requests + placed results + group_first | statuses | calls | out | request results | frames]
    const uint64_t runs = (uint64_t)c->opt.max_runs;
    SlotLayout L;
    H2ClientRingDev& H = c->h2c_dev;
    H.off_args = sizeof(RingSlotHdr);
    c->ring_dev.off_runs = L.add(runs * sizeof(b2_run));
    c->ring_dev.off_in = L.add((uint64_t)max_bytes + 16);
    H.off_reqs = L.add(h2c_ring_block(max_reqs, max_reqs));
    H.off_rs = L.add(runs * sizeof(b2_h2_run_status));
    H.off_calls = L.add((uint64_t)call_cap * sizeof(b2_h2_call));
    H.off_out = L.add((uint64_t)out_cap + 16);
    H.off_req_res = L.add((uint64_t)max_reqs * sizeof(b2_h2_request_result));
    H.off_req_out = L.add((uint64_t)req_out_cap + 16);
    rc = ring_alloc(c, L.end); if (rc != B2_OK) return rc;
    CU(cudaFuncSetAttribute(k_h2_client_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kH2ClientRingSmem));
    c->h2c_max_bytes = max_bytes; c->h2c_call_cap = call_cap; c->h2c_out_cap = out_cap; c->h2c_max_reqs = max_reqs; c->h2c_req_out_cap = req_out_cap;
    c->ring_kind = RingKind::h2_client;
    return B2_OK;
}
extern "C" int b2_h2_client_ring_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                        const b2_h2_request* reqs, uint32_t n_reqs, uint32_t* ticket) {
    if (!c || !bytes || !ticket || (!runs && n_runs) || (!reqs && n_reqs)) { set_err("null argument"); return B2_E_INVAL; }
    if (n_runs == 0 && n_reqs == 0) { set_err("a ticket carries runs, requests or both"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::h2_client) { set_err("b2_h2_client_ring_enable first"); return B2_E_INVAL; }
    // the argument checks of b2_h2_client_process_batch and b2_h2_pack_requests with the caps of b2_h2_client_ring_enable
    if (nbytes > c->h2c_max_bytes) { set_err("ticket larger than b2_h2_client_ring_enable's max_bytes: use the batch calls"); return B2_E_CAPACITY; }
    if (n_runs > c->opt.max_runs || n_reqs > c->h2c_max_reqs) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    H2Split sp = { 0, 0, 0, true };
    if (n_runs) {
        if (!h2_runs_ok(c, runs, n_runs, nbytes)) return B2_E_INVAL;
        sp = h2_split(c->h2c_out_cap, c->h2c_call_cap, 0, n_runs);
        if (!sp.fits) { set_err("out_cap / call_cap too small for the number of runs"); return B2_E_CAPACITY; }
    }
    uint8_t* slot = ring_claim(c, "b2_h2_client_ring_wait");
    if (!slot) return B2_E_CAPACITY;
    std::vector<uint32_t> first;
    std::vector<b2_h2_request_result> placed(n_reqs);
    uint64_t total = 0;
    if (n_reqs) { int rc = h2_place_requests(c, bytes, nbytes, reqs, n_reqs, c->h2c_req_out_cap, placed.data(), first, total); if (rc != B2_OK) return rc; }
    const H2ClientRingArgs a = { sp.per_run, sp.region, n_runs && h2_gz_wanted(c, runs, n_runs) ? 1u : 0u, n_reqs, n_reqs ? (uint32_t)first.size() - 1 : 0u, { 0, 0, 0 } };
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    uint8_t* block = slot + c->h2c_dev.off_reqs;                 // the request block the kernel pulls: requests, placed results, group_first
    if (n_reqs) {
        memcpy(block, reqs, sizeof(b2_h2_request) * (size_t)n_reqs);
        memcpy(block + h2c_ring_res_off(n_reqs), placed.data(), sizeof(b2_h2_request_result) * (size_t)n_reqs);
        memcpy(block + h2c_ring_first_off(n_reqs), first.data(), 4 * first.size());
    }
    memcpy(slot + c->h2c_dev.off_args, &a, sizeof a);
    return ring_ring(c, h, bytes, ticket);
}
extern "C" int b2_h2_client_ring_wait(b2_ctx* c, uint32_t ticket, b2_h2_client_ring_result* out) {
    static_assert(sizeof(b2_h2_client_ring_result) == 64, "h2 client ring result ABI layout");
    int rc;
    const uint8_t* slot = ring_collect(c, c && out && c->ring_kind == RingKind::h2_client, ticket, "bad h2 client ring ticket", rc);
    if (!slot) return rc;
    const RingSlotHdr* h = reinterpret_cast<const RingSlotHdr*>(slot);
    const H2ClientRingDev& L = c->h2c_dev;
    const H2ClientRingArgs* a = reinterpret_cast<const H2ClientRingArgs*>(slot + L.off_args);
    const uint32_t n_runs = h->n_runs;
    const b2_h2_run_status* rs = reinterpret_cast<const b2_h2_run_status*>(slot + L.off_rs);
    uint32_t n_calls = 0;
    for (uint32_t r = 0; r < n_runs; r++) n_calls += rs[r].n_msgs;
    memset(out, 0, sizeof *out);
    out->runs = rs; out->n_runs = n_runs; out->n_calls = n_calls;
    out->calls = reinterpret_cast<const b2_h2_call*>(slot + L.off_calls);
    out->out = slot + L.off_out; out->region = a->region;
    out->n_reqs = a->n_reqs;
    out->reqs = reinterpret_cast<const b2_h2_request_result*>(slot + L.off_req_res);
    out->req_out = slot + L.off_req_out;
    return B2_OK;
}

// ---- baidu_std turns on the latency path: k_ring<RingBody::requests> (b2_client_ring_*) and k_ring<RingBody::replies> (b2_ring_turn_*)
// on the same submit ring (include/b2rpc.h).  Both kinds pack one record per warp after the runs; they differ in the record and in what
// checks and places it (place_requests / place_replies).
struct PackRingNames { const char *enable, *submit, *wait, *recs, *max_recs; };
static const PackRingNames kClientRing = { "b2_client_ring_enable", "b2_client_ring_submit", "b2_client_ring_wait", "requests", "max_reqs" };
static const PackRingNames kTurnRing = { "b2_ring_turn_enable", "b2_ring_turn_submit", "b2_ring_turn_wait", "replies", "max_resps" };
static int pack_ring_enable(b2_ctx* c, RingKind kind, const PackRingNames& nm, uint32_t max_bytes, uint32_t max_recs, uint32_t rec_bytes, uint32_t out_cap) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::none) { set_err("%s: once, before the context's first ring call, and not with another ring kind", nm.enable); return B2_E_INVAL; }
    if (c->has_streams) { set_err("%s: the ticket runs no stream pass, so not on a context with a stream table", nm.enable); return B2_E_INVAL; }
    if (max_bytes == 0 || max_recs == 0 || out_cap == 0) { set_err("capacities must be non-zero"); return B2_E_INVAL; }
    // the limits of b2_process_batch and of the batch pack call, both of which read the ticket's bytes; the records land in d_msgs
    if (max_bytes > c->opt.max_batch_bytes || (uint64_t)max_recs * rec_bytes > (uint64_t)c->opt.max_msgs * 64 || out_cap > c->opt.max_resp_bytes) {
        set_err("exceeds ctx capacity"); return B2_E_CAPACITY;
    }
    CU(cudaSetDevice(c->opt.device));
    static_assert(sizeof(RingSlotHdr) + sizeof(PackRingArgs) <= 256, "pack ring slot header");
    // [RingSlotHdr | args | runs | staged input | records + placed offsets | compact block | frame lengths | frames]
    SlotLayout L;
    PackRingDev& Q = c->pr_dev;
    Q.off_args = sizeof(RingSlotHdr);
    c->ring_dev.off_runs = L.add(kSmallRuns * sizeof(b2_run));
    c->ring_dev.off_in = L.add((uint64_t)max_bytes + 16);
    Q.off_recs = L.add((uint64_t)max_recs * (rec_bytes + 4) + 16);      // (+16: the kernel pulls the records in whole 16-byte words)
    c->ring_dev.off_out = L.add(kSmallBlock);
    Q.off_lens = L.add((uint64_t)max_recs * 4);
    Q.off_out = L.add((uint64_t)out_cap + 16);
    int rc = ring_alloc(c, L.end); if (rc != B2_OK) return rc;
    if (kind == RingKind::batch_client) CU(cudaFuncSetAttribute(k_ring<RingBody::requests>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallSmem)));
    else CU(cudaFuncSetAttribute(k_ring<RingBody::replies>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallSmem)));
    c->pr_max_bytes = max_bytes; c->pr_max_recs = max_recs; c->pr_out_cap = out_cap;
    c->ring_kind = kind;
    return B2_OK;
}
// place(block + n_recs * rec_bytes, total): the kind's checks of its records, and their offsets placed right behind them in the slot
template <class Place>
static int pack_ring_submit(b2_ctx* c, RingKind kind, const PackRingNames& nm, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                            const void* recs, uint32_t n_recs, size_t rec_bytes, Place place, uint32_t* ticket) {
    if (!c || !bytes || !ticket || (!runs && n_runs) || (!recs && n_recs)) { set_err("null argument"); return B2_E_INVAL; }
    if (n_runs == 0 && n_recs == 0) { set_err("a ticket carries runs, %s or both", nm.recs); return B2_E_INVAL; }
    if (c->ring_kind != kind) { set_err("%s first", nm.enable); return B2_E_INVAL; }
    // the argument checks of b2_ring_submit and of the batch pack call with the enable-time caps
    if (nbytes > c->pr_max_bytes) { set_err("ticket larger than %s's max_bytes: use the batch calls", nm.enable); return B2_E_CAPACITY; }
    if (n_runs > kSmallRuns || n_runs > c->opt.max_runs) { set_err("%s serves up to 512 runs: use the batch calls", nm.submit); return B2_E_CAPACITY; }
    if (n_recs > c->pr_max_recs) { set_err("more %s than the enable call's %s", nm.recs, nm.max_recs); return B2_E_CAPACITY; }
    uint8_t* slot = ring_claim(c, nm.wait);
    if (!slot) return B2_E_CAPACITY;
    uint32_t extent = 0;                                         // (the compact block is sized for the bytes the runs cover)
    for (uint32_t r = 0; r < n_runs; r++) {
        if ((runs[r].offset & 15u) || (uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run offset must be 16-aligned and inside the batch"); return B2_E_INVAL; }
        extent = std::max(extent, runs[r].offset + runs[r].length);
    }
    uint8_t* block = slot + c->pr_dev.off_recs;                  // the record block the kernel pulls: records, then their placed offsets
    uint64_t total = 0;
    int rc = place(reinterpret_cast<uint32_t*>(block + rec_bytes * n_recs), total);
    if (rc != B2_OK) return rc;
    if (n_recs) memcpy(block, recs, rec_bytes * n_recs);
    const PackRingArgs a = { n_recs, { 0, 0, 0 } };
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    ring_compact(c, h, small_layout(std::min(extent, kSmallBytes), n_runs, c->opt.max_msgs));
    memcpy(slot + c->pr_dev.off_args, &a, sizeof a);
    return ring_ring(c, h, bytes, ticket);
}
// the runs' result (an overflowing ticket's runs go through the big pipeline here) and views of the ticket's frames in its slot: out's
// batch, then its count, offsets, lengths and frames (the members named)
template <class Result>
static int pack_ring_wait(b2_ctx* c, RingKind kind, const char* bad_ticket, uint32_t ticket, size_t rec_bytes, Result* out, uint32_t Result::*n_recs,
                          const uint32_t* Result::*offs, const uint32_t* Result::*lens, const uint8_t* Result::*frames) {
    int rc;
    uint8_t* slot = ring_collect(c, c && out && c->ring_kind == kind, ticket, bad_ticket, rc);
    if (!slot) return rc;
    memset(out, 0, sizeof *out);
    const PackRingDev& L = c->pr_dev;
    const uint32_t n = reinterpret_cast<const PackRingArgs*>(slot + L.off_args)->n_recs;
    out->*n_recs = n;
    out->*offs = reinterpret_cast<const uint32_t*>(slot + L.off_recs + rec_bytes * n);
    out->*lens = reinterpret_cast<const uint32_t*>(slot + L.off_lens);
    out->*frames = slot + L.off_out;
    return ring_batch_result(c, ticket, slot, &out->batch);
}

extern "C" int b2_client_ring_enable(b2_ctx* c, uint32_t max_bytes, uint32_t max_reqs, uint32_t req_out_cap) {
    return pack_ring_enable(c, RingKind::batch_client, kClientRing, max_bytes, max_reqs, sizeof(b2_request), req_out_cap);
}
extern "C" int b2_client_ring_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                     const b2_request* reqs, uint32_t n_reqs, uint32_t* ticket) {
    return pack_ring_submit(c, RingKind::batch_client, kClientRing, bytes, nbytes, runs, n_runs, reqs, n_reqs, sizeof(b2_request),
                            [&](uint32_t* offs, uint64_t& total) { return place_requests(nbytes, reqs, n_reqs, c->pr_out_cap, offs, total); }, ticket);
}
extern "C" int b2_client_ring_wait(b2_ctx* c, uint32_t ticket, b2_client_ring_result* out) {
    static_assert(sizeof(b2_client_ring_result) == 104, "client ring result ABI layout");
    return pack_ring_wait(c, RingKind::batch_client, "bad client ring ticket", ticket, sizeof(b2_request), out, &b2_client_ring_result::n_reqs,
                          &b2_client_ring_result::req_offs, &b2_client_ring_result::req_lens, &b2_client_ring_result::req_out);
}
extern "C" int b2_ring_turn_enable(b2_ctx* c, uint32_t max_bytes, uint32_t max_resps, uint32_t resp_out_cap) {
    return pack_ring_enable(c, RingKind::batch_replies, kTurnRing, max_bytes, max_resps, sizeof(b2_reply), resp_out_cap);
}
extern "C" int b2_ring_turn_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                   const b2_reply* replies, uint32_t n_replies, uint32_t* ticket) {
    return pack_ring_submit(c, RingKind::batch_replies, kTurnRing, bytes, nbytes, runs, n_runs, replies, n_replies, sizeof(b2_reply),
                            [&](uint32_t* offs, uint64_t& total) { return place_replies(bytes, nbytes, replies, n_replies, c->pr_out_cap, offs, total); }, ticket);
}
extern "C" int b2_ring_turn_wait(b2_ctx* c, uint32_t ticket, b2_ring_turn_result* out) {
    static_assert(sizeof(b2_ring_turn_result) == 104, "ring turn result ABI layout");
    return pack_ring_wait(c, RingKind::batch_replies, "bad ring turn ticket", ticket, sizeof(b2_reply), out, &b2_ring_turn_result::n_replies,
                          &b2_ring_turn_result::reply_offs, &b2_ring_turn_result::reply_lens, &b2_ring_turn_result::reply_out);
}

// ---- a Stream producer's turn on the latency path: k_ring<RingBody::stream_writes> (include/b2rpc.h, b2_stream_ring_write_enable) ----
extern "C" int b2_stream_ring_write_enable(b2_ctx* c, uint32_t max_bytes, uint32_t max_writes, uint32_t write_out_cap, uint32_t max_segment_size) {
    if (!c) { set_err("null argument"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::batch_streams || c->ring_slots) { set_err("b2_stream_ring_write_enable: after b2_stream_ring_enable and before the context's first ring call"); return B2_E_INVAL; }
    if (max_bytes == 0 || max_writes == 0 || write_out_cap == 0) { set_err("capacities must be non-zero"); return B2_E_INVAL; }
    // the limits of b2_process_batch and b2_stream_write, both of which read the ticket's bytes
    if (max_bytes > c->opt.max_batch_bytes || max_writes > c->opt.max_msgs || write_out_cap > c->opt.max_resp_bytes) { set_err("exceeds ctx capacity"); return B2_E_CAPACITY; }
    CU(cudaSetDevice(c->opt.device));
    static_assert(sizeof(RingSlotHdr) + sizeof(SwRingArgs) <= 256, "stream write ring slot header");
    int rc = sw_host_recs(c, max_writes);               // (the records are resolved there before they go into the slot)
    if (rc != B2_OK) return rc;
    // the write pass's scratch, as sw_launch lays out d_sw[2] / d_sw[3] / d_sw[1] for a call of max_writes writes
    const size_t mw = max_writes, cap = c->sp.cap;
    const size_t o_res = (mw * 24 + 15) & ~(size_t)15, o_slot = o_res + 32 * mw, o_group = o_slot + ((4 * mw + 15) & ~(size_t)15),
                 o_fb = o_group + 8 * mw, o_cb = o_fb + ((4 * mw + 15) & ~(size_t)15), o_ps = (o_cb + 4 * mw + 255) & ~(size_t)255,
                 o_out = (o_ps + 64 + 16 * cap + 255) & ~(size_t)255;
    cudaFree(c->d_swr); c->d_swr = nullptr;
    if (cudaMalloc((void**)&c->d_swr, o_out + write_out_cap + 32) != cudaSuccess) { cudaGetLastError(); set_err("cudaMalloc of the stream write ring scratch failed"); return B2_E_NOMEM; }
    CU(cudaMemset(c->d_swr + o_ps, 0, 64 + 16 * cap));  // counters | cnt | fill: the ring's tickets start from zeros
    SwPass& P = c->swr_dev.pass;
    P.tab = c->sp.tab; P.cap = c->sp.cap; P.recs = reinterpret_cast<const SwRec*>(c->d_swr); P.n = 0;
    P.seg = max_segment_size ? max_segment_size : 512u << 20;                     // -stream_write_max_segment_size (stream.cpp:39)
    uint32_t* per_slot = reinterpret_cast<uint32_t*>(c->d_swr + o_ps);
    P.cnts = per_slot; P.cnt = per_slot + 16; P.fill = P.cnt + cap; P.base = P.fill + cap; P.touched = P.base + cap;
    P.res = reinterpret_cast<b2_stream_write_result*>(c->d_swr + o_res); P.slot = reinterpret_cast<uint32_t*>(c->d_swr + o_slot);
    P.group = reinterpret_cast<uint32_t*>(c->d_swr + o_group); P.frame_base = reinterpret_cast<uint32_t*>(c->d_swr + o_fb);
    P.chunk_base = reinterpret_cast<uint32_t*>(c->d_swr + o_cb); P.out = c->d_swr + o_out;
    // [RingSlotHdr | args | runs | staged input | write records | compact block | stream section | write results | frames]
    SlotLayout L;
    SwRingDev& Q = c->swr_dev;
    RingDev& R = c->ring_dev;
    Q.off_args = sizeof(RingSlotHdr);
    R.off_runs = L.add(kSmallRuns * sizeof(b2_run));
    R.off_in = L.add((uint64_t)max_bytes + 16);
    Q.off_recs = L.add(mw * sizeof(SwRec) + 16);
    R.off_out = L.add(kSmallBlock);
    R.off_st = L.add(kSecOut + ((c->sp_ring.out_cap + 15u) & ~15u));
    Q.off_res = L.add(mw * sizeof(b2_stream_write_result) + 16);
    Q.off_wout = L.add((uint64_t)write_out_cap + 16);
    if ((rc = ring_alloc(c, L.end)) != B2_OK) return rc;
    CU(cudaFuncSetAttribute(k_ring<RingBody::stream_writes>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallSmem)));
    c->swr_max_bytes = max_bytes; c->swr_max_writes = max_writes; c->swr_out_cap = write_out_cap;
    c->ring_kind = RingKind::batch_stream_writes;
    return B2_OK;
}
extern "C" int b2_stream_ring_submit(b2_ctx* c, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                     const b2_stream_write_desc* writes, uint32_t n_writes, uint32_t* ticket) {
    if (!c || !bytes || !ticket || (!runs && n_runs) || (!writes && n_writes)) { set_err("null argument"); return B2_E_INVAL; }
    if (n_runs == 0 && n_writes == 0) { set_err("a ticket carries runs, writes or both"); return B2_E_INVAL; }
    if (c->ring_kind != RingKind::batch_stream_writes) { set_err("b2_stream_ring_write_enable first"); return B2_E_INVAL; }
    // the argument checks of b2_ring_submit and b2_stream_write with the caps of b2_stream_ring_write_enable
    if (nbytes > c->swr_max_bytes) { set_err("ticket larger than b2_stream_ring_write_enable's max_bytes: use the batch calls"); return B2_E_CAPACITY; }
    if (n_runs > kSmallRuns || n_runs > c->opt.max_runs) { set_err("b2_stream_ring_submit serves up to 512 runs: use the batch calls"); return B2_E_CAPACITY; }
    if (n_writes > c->swr_max_writes) { set_err("more writes than b2_stream_ring_write_enable's max_writes"); return B2_E_CAPACITY; }
    uint8_t* slot = ring_claim(c, "b2_stream_ring_wait");
    if (!slot) return B2_E_CAPACITY;
    uint32_t extent = 0;                                         // (the compact block is sized for the bytes the runs cover)
    for (uint32_t r = 0; r < n_runs; r++) {
        if ((runs[r].offset & 15u) || (uint64_t)runs[r].offset + runs[r].length > nbytes) { set_err("run offset must be 16-aligned and inside the batch"); return B2_E_INVAL; }
        extent = std::max(extent, runs[r].offset + runs[r].length);
    }
    // the kernel pulls every ticket into d_bytes: that is where a host-sourced payload is
    uint64_t bound = 0;
    int rc = sw_resolve(c, writes, n_writes, nbytes, c->swr_dev.pass.seg, c->d_bytes, false, c->h_sw_recs, bound);
    if (rc != B2_OK) return rc;
    if (bound > c->swr_out_cap) { set_err("write_out_cap below the sum of align16(len + ceil(len / seg) * 38)"); return B2_E_CAPACITY; }
    const SwRingArgs a = { n_writes, (uint32_t)bound, { 0, 0 } };
    RingSlotHdr* h = ring_fill(c, slot, bytes, nbytes, runs, n_runs);
    ring_compact(c, h, small_layout(std::min(extent, kSmallBytes), n_runs, c->opt.max_msgs));
    if (n_writes) memcpy(slot + c->swr_dev.off_recs, c->h_sw_recs, sizeof(SwRec) * (size_t)n_writes);
    memcpy(slot + c->swr_dev.off_args, &a, sizeof a);
    return ring_ring(c, h, bytes, ticket);
}
extern "C" int b2_stream_ring_wait(b2_ctx* c, uint32_t ticket, b2_stream_ring_result* out) {
    static_assert(sizeof(b2_stream_ring_result) == 96, "stream ring result ABI layout");
    int rc;
    uint8_t* slot = ring_collect(c, c && out && c->ring_kind == RingKind::batch_stream_writes, ticket, "bad stream ring ticket", rc);
    if (!slot) return rc;
    memset(out, 0, sizeof *out);
    const SwRingDev& L = c->swr_dev;
    const SwRingArgs args = *reinterpret_cast<const SwRingArgs*>(slot + L.off_args);
    const uint32_t n = args.n_writes;
    b2_stream_write_result* res = reinterpret_cast<b2_stream_write_result*>(slot + L.off_res);
    const bool overflow = reinterpret_cast<const uint32_t*>(slot + c->ring_dev.off_out)[2] & 3u;
    rc = ring_batch_result(c, ticket, slot, &out->batch, false);
    if (overflow) {
        // k_ring ran neither pass and parks behind the ticket: the big pipeline has served the runs (and their stream pass); the writes go
        // through the grid path on the ticket's own bytes, and only then does the next ticket see the table
        if (rc == B2_OK && n) {
            const SwRec* recs = reinterpret_cast<const SwRec*>(slot + L.off_recs);
            uint32_t used = 0;
            rc = sw_reserve(c, 0, reinterpret_cast<const RingSlotHdr*>(slot)->nbytes);
            if (rc == B2_OK) {
                const uint8_t* d_in = static_cast<const uint8_t*>(c->d_sw[0]);      // (the staging the grid path copies the bytes into)
                for (uint32_t i = 0; i < n; i++) { c->h_sw_recs[i] = recs[i]; c->h_sw_recs[i].src = d_in + (recs[i].src - c->d_bytes); }
                rc = sw_launch(c, c->ring_bytes[ticket % kRingSlots], reinterpret_cast<const RingSlotHdr*>(slot)->nbytes, n, L.pass.seg, args.bound, res,
                               slot + L.off_wout, &used);
            }
        }
        ring_unpark(c, ticket);
        if (rc != B2_OK) return rc;
    }
    if (rc != B2_OK) return rc;
    uint32_t used = 0;                                           // (out_off grows in array order; the gaps are part of the frames)
    for (uint32_t i = 0; i < n; i++) used = std::max(used, res[i].out_off + ((res[i].out_len + 15u) & ~15u));
    out->n_writes = n; out->out_bytes = used;
    out->results = res; out->out = slot + L.off_wout;
    return B2_OK;
}
