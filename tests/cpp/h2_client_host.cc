// Test harness (not product): the client side of brpc_b200/csrc/b2_h2.cuh — k_h2_client_conn_reset, k_h2_pack_req, k_h2_client_consume,
// k_h2_client_abandon — built for the host on top of the harness tests/cpp/gen_h2_host.py writes (h2_host.cc: the device source as it
// stands, a "warp" of one thread), laid out the way brpc_b200/csrc/b2_api.cu lays the device side out.  Adds a snapshot of one connection's
// state so that one byte stream can be cut at every offset without replaying what came before, and the every-offset comparison itself.
#include "h2_host.cc"
#include <string>
#include <vector>

extern "C" {
void h2c_client_reset(h2h_ctx* c, uint32_t conn) { blockDim.x = 1; blockIdx.x = 0; threadIdx.x = 0; k_h2_client_conn_reset(c->conns, c->hps, conn, pool_of(c)); }
void h2c_abandon(h2h_ctx* c, uint32_t conn, const uint32_t* ids, uint32_t n) { blockDim.x = 1; blockIdx.x = 0; threadIdx.x = 0; k_h2_client_abandon(c->conns, conn, ids, n, pool_of(c)); }
// b2_h2_pack_requests around the kernel: group_first[0..n_groups] as the API builds it, results[i].out_off filled by the caller
void h2c_pack(h2h_ctx* c, const uint8_t* bytes, const b2_h2_request* reqs, const uint32_t* group_first, uint32_t n_groups, uint8_t* out,
              b2_h2_request_result* results) {
    blockDim.x = kH2PackWarps * 32;
    for (uint32_t g = 0; g < n_groups; g++) {
        blockIdx.x = g / kH2PackWarps; threadIdx.x = (g % kH2PackWarps) * 32;            // lane 0 of warp g
        k_h2_pack_req(bytes, reqs, group_first, n_groups, c->conns, out, results, pool_of(c));
    }
}
// b2_h2_client_process_batch around the kernel: every run owns `region` bytes of out and per_run_calls descriptors
void h2c_consume(h2h_ctx* c, const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, b2_h2_run_status* rs, b2_h2_call* calls,
                 uint32_t per_run_calls, uint8_t* out, uint32_t region) {
    blockDim.x = 1; threadIdx.x = 0;
    for (uint32_t r = 0; r < n_runs; r++) { blockIdx.x = r; k_h2_client_consume(bytes, runs, n_runs, c->conns, c->hps, rs, calls, per_run_calls, out, region, pool_of(c)); }
}

// ---- one connection's state, saved and put back (the live streams' header records and copied bodies only)
struct h2c_snap { H2Conn conn; HpackState hp; std::vector<H2Stream> S; std::vector<std::string> hdr, body; };
void* h2c_snapshot(h2h_ctx* c, uint32_t conn) {
    h2c_snap* s = new h2c_snap;
    const uint32_t P = c->pending;
    s->conn = c->conns[conn]; s->hp = c->hps[conn];
    s->S.assign(c->streams + (size_t)conn * P, c->streams + (size_t)(conn + 1) * P);
    s->hdr.resize(P); s->body.resize(P);
    for (uint32_t k = 0; k < P; k++) if (s->S[k].id >= 0) {
        const uint8_t* slot = c->slots + ((size_t)conn * P + k) * c->stream_bytes;
        s->hdr[k].assign((const char*)slot, s->S[k].hdr_len);
        if (!s->S[k].body_input_off) s->body[k].assign((const char*)slot + kH2HdrBytes, s->S[k].body_len);
    }
    return s;
}
void h2c_restore(h2h_ctx* c, uint32_t conn, void* snap) {
    const h2c_snap* s = (const h2c_snap*)snap;
    const uint32_t P = c->pending;
    c->conns[conn] = s->conn; c->hps[conn] = s->hp;
    memcpy(c->streams + (size_t)conn * P, s->S.data(), sizeof(H2Stream) * P);
    for (uint32_t k = 0; k < P; k++) if (s->S[k].id >= 0) {
        uint8_t* slot = c->slots + ((size_t)conn * P + k) * c->stream_bytes;
        memcpy(slot, s->hdr[k].data(), s->hdr[k].size());
        memcpy(slot + kH2HdrBytes, s->body[k].data(), s->body[k].size());
    }
}
void h2c_snap_free(void* snap) { delete (h2c_snap*)snap; }

// ---- what a run produced, without the places it was put: parse error, ctrl bytes, every call's fields and the bytes they point at
struct h2c_scratch { std::vector<uint8_t> in, out; std::vector<b2_h2_call> calls; };
// (ctrl bytes and calls go to two strings: a cut moves calls and acks between the two runs independently)
static uint32_t run_once(h2h_ctx* c, uint32_t conn, h2c_scratch& x, const std::string& bytes, uint32_t region, uint32_t cap, std::string& canon, std::string& ctrl) {
    x.in.assign(bytes.begin(), bytes.end()); x.in.resize(bytes.size() + 64, 0);
    x.out.assign(region, 0); x.calls.assign(cap, b2_h2_call());
    b2_run run; memset(&run, 0, sizeof run); run.socket_id = conn; run.offset = 0; run.length = (uint32_t)bytes.size();
    b2_h2_run_status rs;
    h2c_consume(c, x.in.data(), &run, 1, &rs, x.calls.data(), cap, x.out.data(), region);
    ctrl.append((const char*)x.out.data() + rs.ctrl_off, rs.ctrl_len);
    for (uint32_t i = 0; i < rs.n_msgs; i++) {
        const b2_h2_call& m = x.calls[i];
        int32_t f[7] = { (int32_t)m.stream_id, (int32_t)m.how, m.status_code, m.error_code, m.grpc_status, (int32_t)m.flags, (int32_t)m.n_headers };
        canon.append("|call", 5); canon.append((const char*)f, sizeof f);
        const uint8_t* src = (m.flags & B2_H2_FLAG_BODY_IN_INPUT) ? x.in.data() : x.out.data();
        canon.append((const char*)x.out.data() + m.headers_off, m.headers_len); canon.push_back('|');
        canon.append((const char*)src + m.body_off, m.body_len); canon.push_back('|');
        canon.append((const char*)src + m.msg_off, m.msg_len); canon.push_back('|');
        canon.append((const char*)x.out.data() + m.error_off, m.error_len); canon.push_back('|');
    }
    if (rs.parse_error != B2_PARSE_ERROR_NOT_ENOUGH_DATA) { canon.append("|error", 6); canon.push_back((char)rs.parse_error); }
    return rs.parse_error == B2_PARSE_ERROR_NOT_ENOUGH_DATA ? rs.consumed : 0xffffffffu;
}
// `rest` (bytes left over from before) + seg[0, len) parsed whole, and again cut at every offset `step` apart into two runs (the second
// one starts with what the first left unconsumed); each cut must give the same ctrl bytes, calls and leftover.  The connection is left
// as the whole parse leaves it; *left_len = its leftover length.  Returns the number of cuts that differed (*first_bad: the first).
uint32_t h2c_every_offset(h2h_ctx* c, uint32_t conn, const uint8_t* rest, uint32_t rest_len, const uint8_t* seg, uint32_t len, uint32_t step,
                          uint32_t region, uint32_t cap, uint32_t* first_bad, uint32_t* n_cuts, uint32_t* left_len) {
    h2c_scratch x;
    void* snap = h2c_snapshot(c, conn);
    const std::string whole = std::string((const char*)rest, rest_len) + std::string((const char*)seg, len);
    std::string want, want_ctrl;
    const uint32_t used = run_once(c, conn, x, whole, region, cap, want, want_ctrl);
    if (used != 0xffffffffu) want.append("|left", 5), want.append(whole, used, std::string::npos);
    uint32_t bad = 0, cuts = 0; *first_bad = 0xffffffffu;
    for (uint32_t cut = 0; cut <= len; cut += step) {
        h2c_restore(c, conn, snap);
        std::string got, got_ctrl;
        const std::string a = std::string((const char*)rest, rest_len) + std::string((const char*)seg, cut);
        const uint32_t u1 = run_once(c, conn, x, a, region, cap, got, got_ctrl);
        if (u1 != 0xffffffffu) {
            const std::string b = a.substr(u1) + std::string((const char*)seg + cut, len - cut);
            const uint32_t u2 = run_once(c, conn, x, b, region, cap, got, got_ctrl);
            if (u2 != 0xffffffffu) got.append("|left", 5), got.append(b, u2, std::string::npos);
        }
        cuts++;
        if (got != want || got_ctrl != want_ctrl) { if (!bad) *first_bad = cut; bad++; }
    }
    h2c_restore(c, conn, snap);
    std::string again, again_ctrl;
    (void)run_once(c, conn, x, whole, region, cap, again, again_ctrl);
    h2c_snap_free(snap);
    *n_cuts = cuts; *left_len = used == 0xffffffffu ? 0 : (uint32_t)whole.size() - used;
    return bad;
}
}
