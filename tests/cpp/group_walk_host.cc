// Test harness (not product): the group walk of k_tile_walk (B.walk_group > 1) from the generated host-compilable copy of
// brpc_b200/csrc/b2_kernels.cuh (tests/cpp/gen_kernels_host.py), one thread per group, then k_resolve and k_frame_table as kh_front
// (decode_host.cc) runs them; and the per-tile k_tile_walk from every member's entry, to compare the records member by member.
#include "kernels_host_prelude.h"
#include "kernels_host.cuh"
#include <vector>
using namespace b2;
namespace b2 { __attribute__((aligned(128))) uint8_t fused_raw[16], pack_smem_raw[16], small_raw[16]; __attribute__((aligned(16))) uint8_t s_rings[16]; uint32_t sm[4]; }

namespace {
struct Front {
    std::vector<uint32_t> rtb, heads, tile_base, scratch, spec, totals;
    std::vector<uint4> ti;
    std::vector<TileRec> tiles, head_recs;
    BatchPtrs B;
    DevConfig C;
    uint32_t nt = 0;
    Front(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, uint32_t tile_shift, uint32_t proto_mask, uint64_t max_body, uint32_t group) {
        const uint32_t tile = 1u << tile_shift;
        rtb.assign(n_runs + 1, 0);
        for (uint32_t r = 0; r < n_runs; r++) rtb[r + 1] = rtb[r] + (uint32_t)(((uint64_t)runs[r].length + tile - 1) >> tile_shift);
        nt = rtb[n_runs];
        ti.resize(nt ? nt : 1);
        for (uint32_t r = 0; r < n_runs; r++) {
            for (uint32_t t = rtb[r]; t < rtb[r + 1]; t++) ti[t] = make_uint4(runs[r].offset, runs[r].length, t - rtb[r], r | (runs[r].flags << 24));
            for (uint32_t t = rtb[r]; t < rtb[r + 1]; t += group) heads.push_back(t);          // (what b2_batch_upload lays out)
        }
        if (heads.empty()) heads.push_back(0);
        tiles.resize(nt ? nt : 1); tile_base.assign(nt + 1, 0); scratch.assign(3 * (size_t)nt + 3, 0); spec.assign((size_t)kSpecK * nt + 1, 0); totals.assign(16, 0);
        memset(&B, 0, sizeof B);
        B.bytes = bytes; B.runs = runs; B.run_tile_base = rtb.data(); B.tile_info = ti.data(); B.tiles = tiles.data(); B.tile_base = tile_base.data();
        B.tile_scratch = scratch.data(); B.tile_spec = spec.data(); B.totals = totals.data();
        B.n_runs = n_runs; B.n_tiles = nt; B.max_resp = 0xfffffff0u;
        head_recs.resize(heads.size());
        B.group_heads = heads.data(); B.head_recs = head_recs.data(); B.n_groups = group > 1 ? (uint32_t)heads.size() : 0; B.walk_group = group;
        memset(&C, 0, sizeof C);
        C.max_body_size = max_body ? max_body : (64ull << 20); C.tile_bytes = tile; C.tile_shift = tile_shift; C.spec_k = kSpecK; C.proto_mask = proto_mask;
        blockDim.x = 1; threadIdx.x = 0; gridDim.x = 0x7fffffffu;            // (the last-CTA epilogues never fire)
    }
    // k_tile_walk over every group (group > 1) or every tile; `entries` holds every tile's speculative entry (grouped: only the heads'
    // are used, handed over in head_recs as k_tile_search leaves them)
    void walk(const uint32_t* entries) {
        for (uint32_t t = 0; t < nt; t++) { memset(&tiles[t], 0, sizeof(TileRec)); tiles[t].entry = B.walk_group > 1 ? 0xdeadbeefu : entries[t]; }
        for (size_t g = 0; g < head_recs.size(); g++) { memset(&head_recs[g], 0, sizeof(TileRec)); head_recs[g].entry = entries[heads[g]]; }
        const uint32_t n = B.walk_group > 1 ? B.n_groups : nt;
        for (uint32_t i = 0; i < n; i++) { blockIdx.x = i; k_tile_walk(B, C); }
    }
};
}

extern "C" {
// The group walk -> k_resolve -> k_frame_table, as kh_front does with the per-tile walk.
int kh_front_group(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, uint32_t tile_shift, uint32_t proto_mask, uint64_t max_body,
                   uint32_t group, const uint32_t* entries, uint32_t n_tiles_expected,
                   b2_run_status* rs_out, uint32_t* frame_off, uint32_t* frame_run, uint32_t cap, uint32_t* n_msgs_out, uint32_t* n_rewalked) {
    Front f(bytes, runs, n_runs, tile_shift, proto_mask, max_body, group);
    if (f.nt != n_tiles_expected) return -1;
    f.B.run_status = rs_out; f.B.frame_off = frame_off; f.B.frame_run = frame_run; f.B.max_msgs = cap;
    f.walk(entries);
    for (uint32_t r = 0; r < n_runs; r++) { blockIdx.x = r; k_resolve(f.B, f.C, 1u); }
    uint32_t total = 0, rew = 0;
    for (uint32_t r = 0; r < n_runs; r++) { rs_out[r].first_msg = total; total += rs_out[r].n_msgs; }
    for (uint32_t t = 0; t < f.nt; t++) rew += (f.tiles[t].kind & kKindRewalked) ? 1u : 0u;
    f.totals[0] = total;
    *n_msgs_out = total; *n_rewalked = rew;
    if (total > cap) return -2;
    for (uint32_t g = 0; g < f.nt * kSpecK; g++) { blockIdx.x = g; k_frame_table(f.B, f.C); }
    return 0;
}

// The group walk's records against the per-tile walk entered at every member's entry.  recs: per tile {entry, exit, count, kind,
// last_proto} of the group walk; returns the number of members whose record or offsets differ (-1 on a shape mismatch), *n_entered the
// number of members the group walk entered.
int kh_group_vs_tiles(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, uint32_t tile_shift, uint32_t proto_mask, uint64_t max_body,
                      uint32_t group, const uint32_t* entries, uint32_t n_tiles_expected, uint32_t* recs, uint32_t* n_entered) {
    Front g(bytes, runs, n_runs, tile_shift, proto_mask, max_body, group), p(bytes, runs, n_runs, tile_shift, proto_mask, max_body, 1);
    if (g.nt != n_tiles_expected) return -1;
    g.walk(entries);
    std::vector<uint32_t> member_entries(g.nt + 1);
    for (uint32_t t = 0; t < g.nt; t++) member_entries[t] = g.tiles[t].entry;
    p.walk(member_entries.data());
    int bad = 0; uint32_t entered = 0;
    for (uint32_t t = 0; t < g.nt; t++) {
        const TileRec &a = g.tiles[t], &b = p.tiles[t];
        uint32_t* q = recs + 5 * (size_t)t;
        q[0] = a.entry; q[1] = a.exit; q[2] = a.count; q[3] = a.kind; q[4] = (uint32_t)(int)a.last_proto;
        if (a.entry == kNone) continue;
        entered++;
        bool same = a.exit == b.exit && a.count == b.count && a.kind == b.kind && a.last_proto == b.last_proto && a.live == b.live && a.pf_in == b.pf_in;
        for (uint32_t i = 0; same && i < a.count && i < kSpecK; i++) same = g.spec[(size_t)t * kSpecK + i] == p.spec[(size_t)t * kSpecK + i];
        bad += same ? 0 : 1;
    }
    *n_entered = entered;
    return bad;
}
}
