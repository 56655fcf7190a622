// b2_h2.cuh — h2 frame-head scan and HPACK decode on the device (SURVEY §2.3 K8, §8a a15).
//   h2 frame heads  <- H2Context::ConsumeFrameHead   src/brpc/policy/http2_rpc_protocol.cpp:438-465
//   HPACK decode    <- HPacker::Decode               src/brpc/details/hpack.cpp:765-843 (+ :531-635, :403-473, :72-229)
// Both are per-connection serial state machines (frame chain; dynamic table), so the unit of
// parallelism is the connection: one thread per connection, thousands of connections per batch.
// Further down: ParseH2Message on server and client connections (one frame loop, h2_consume_run, behind k_h2_consume and
// k_h2_client_consume: stream state machine, SETTINGS / WINDOW_UPDATE / GOAWAY side effects as the bytes to write back) and the
// framing of replies (k_h2_pack) and requests (k_h2_pack_req) with HPACK encoding.
#pragma once
#include <cuda_runtime.h>
#include <type_traits>
#include "b2_core.cuh"
#include "b2_hpack_tables.cuh"
#include "b2_inflate.cuh"

namespace b2 {

struct HpackState {                     // one connection's decoder table (IndexTable, hpack.cpp:72-229)
    uint32_t max_size, size, count, head, byte_head, pad[3];
    struct { uint16_t off, nl, vl, pad; } meta[128];   // ring, newest at `head`
    uint8_t bytes[4096];                // ring of name||value bytes, FIFO like the entries
};

#if defined(__CUDACC__)
__device__ __forceinline__ void hp_pop(HpackState& h) {
    const uint32_t i = (h.head + h.count - 1) & 127u;
    h.size -= (uint32_t)h.meta[i].nl + h.meta[i].vl + 32u;
    h.count--;
}
// AddHeader (hpack.cpp:150-177); entry bytes are read from `src` (name then value, contiguous)
__device__ __forceinline__ int hp_add(HpackState& h, const uint8_t* src, uint32_t nl, uint32_t vl) {
    const uint32_t es = nl + vl + 32u;
    if (nl == 0) return -1;                             // reference CHECK-aborts on an empty name
    while (h.count && h.size + es > h.max_size) hp_pop(h);
    if (es > h.max_size) return 0;
    if (h.count >= 128) return -1;
    h.head = (h.head + 127u) & 127u;
    h.meta[h.head].off = (uint16_t)h.byte_head; h.meta[h.head].nl = (uint16_t)nl; h.meta[h.head].vl = (uint16_t)vl;
    for (uint32_t i = 0; i < nl + vl; i++) h.bytes[(h.byte_head + i) & 4095u] = src[i];
    h.byte_head = (h.byte_head + nl + vl) & 4095u;
    h.count++; h.size += es;
    return 0;
}
// DecodeInteger (hpack.cpp:531-565): >0 bytes used, 0 not enough data, -1 malformed
__device__ __forceinline__ int hp_int(const uint8_t* p, uint32_t n, uint32_t prefix, uint32_t& value) {
    if (n == 0) return 0;
    unsigned long long tmp = p[0] & ((1u << prefix) - 1);
    if (tmp < ((1u << prefix) - 1)) { value = (uint32_t)tmp; return 1; }
    uint32_t i = 1; int m = 0; uint8_t cur;
    do {
        if (i >= n) return 0;
        cur = p[i++];
        tmp += (unsigned long long)(cur & 0x7f) << m;
        m += 7;
    } while ((cur & 0x80) && tmp < 10ull * 1024 * 1024);
    if (tmp >= 10ull * 1024 * 1024) return -1;
    value = (uint32_t)tmp;
    return (int)i;
}
// DecodeString (:606-635) with the Huffman walk of HuffmanDecoder (:414-468) over the pre-built tree
__device__ __forceinline__ int hp_str(const uint8_t* p, uint32_t n, uint8_t* out, uint32_t cap, uint32_t& olen) {
    if (n == 0) return 0;
    const bool huffman = p[0] & 0x80;
    uint32_t length = 0;
    const int ib = hp_int(p, n, 7, length);
    if (ib <= 0) return -1;
    if (length > n - (uint32_t)ib) return 0;
    const uint8_t* s = p + ib;
    if (!huffman) {
        if (length > cap) return -2;
        for (uint32_t i = 0; i < length; i++) out[i] = s[i];
        olen = length; return ib + (int)length;
    }
    int node = 0; uint32_t depth = 0, o = 0; bool padding = true;
    for (uint32_t i = 0; i < length; i++) {
        const uint32_t byte = s[i];
        for (int b = 7; b >= 0; b--) {
            const uint32_t bit = (byte >> b) & 1u;
            const int nx = kHuffTree[node][bit];
            if (nx == 0) return -1;                          // NULL_NODE
            if (nx < 0) {
                const int sym = -nx - 1;
                if (sym == 256) return -1;                   // EOS inside the string
                if (o >= cap) return -2;
                out[o++] = (uint8_t)sym; node = 0; depth = 0; padding = true;
                continue;
            }
            node = nx; depth++; padding = padding && bit;
        }
    }
    if (!(depth == 0 || (depth <= 7 && padding))) return -1;
    olen = o; return ib + (int)length;
}
// HeaderAt: 1..61 static, 62.. dynamic newest first; copies name (and value) into out
__device__ __forceinline__ bool hp_copy_indexed(const HpackState& h, uint32_t index, bool with_value, uint8_t* out, uint32_t cap,
                                                uint32_t& nl, uint32_t& vl, bool& overflow) {
    overflow = false;
    if (index >= 1 && index <= 61) {
        nl = kHpackStaticName[index - 1][1]; vl = with_value ? kHpackStaticValue[index - 1][1] : 0;
        if (nl + vl > cap) { overflow = true; return false; }
        for (uint32_t i = 0; i < nl; i++) out[i] = kHpackStaticBlob[kHpackStaticName[index - 1][0] + i];
        for (uint32_t i = 0; i < vl; i++) out[nl + i] = kHpackStaticBlob[kHpackStaticValue[index - 1][0] + i];
        return true;
    }
    if (index >= 62 && index - 62 < h.count) {
        const uint32_t e = (h.head + (index - 62)) & 127u;
        nl = h.meta[e].nl; vl = with_value ? h.meta[e].vl : 0;
        if (nl + vl > cap) { overflow = true; return false; }
        const uint32_t off = h.meta[e].off, nb = nl + vl;
        if (off + nb <= 4096u) {                                      // the entry does not wrap the ring: word copies
            uint32_t i = 0;
            for (; i + 4 <= nb; i += 4) { const uint32_t wv = ld32_any(h.bytes + off + i); out[i] = (uint8_t)wv; out[i + 1] = (uint8_t)(wv >> 8); out[i + 2] = (uint8_t)(wv >> 16); out[i + 3] = (uint8_t)(wv >> 24); }
            for (; i < nb; i++) out[i] = h.bytes[off + i];
        } else for (uint32_t i = 0; i < nb; i++) out[i] = h.bytes[(off + i) & 4095u];
        return true;
    }
    return false;
}
// HPacker::Decode (hpack.cpp:765-843): ONE field at p[0..left).  The record bytes (name then value) land in rec.
// rc > 0: a field was produced, `adv` bytes consumed; rc == 0: ran out of bytes inside an indexed field / size update
// (the iterator is then at the end: the bytes are swallowed, as in the reference); -1 malformed; -2 rec too small.
__device__ __forceinline__ int hpack_decode_field(HpackState& h, const uint8_t* p, uint32_t left, uint8_t* rec, uint32_t cap,
                                                  uint32_t& nl, uint32_t& vl, uint32_t& adv) {
    const uint8_t* p0 = p;
    nl = vl = 0; adv = 0;
    // (001x) dynamic table size updates precede the field they travel with
    while (left && (p[0] >> 5) == 1) {
        uint32_t max_size = 0;
        const int ib = hp_int(p, left, 5, max_size);
        if (ib <= 0) return ib;
        if (max_size > 4096) return -1;
        if (max_size > h.max_size) h.max_size = max_size;
        else if (max_size < h.max_size) { h.max_size = max_size; while (h.size > h.max_size) hp_pop(h); }
        p += ib; left -= (uint32_t)ib;
    }
    if (!left) return 0;
    const uint8_t fb = p[0];
    uint32_t index = 0;
    bool ovf = false;
    if (fb & 0x80) {                                     // indexed field
        const int ib = hp_int(p, left, 7, index);
        if (ib <= 0) return ib;
        if (!hp_copy_indexed(h, index, true, rec, cap, nl, vl, ovf)) return ovf ? -2 : -1;
        p += ib;
    } else {
        const bool incremental = (fb >> 6) == 1;
        const int ib = hp_int(p, left, incremental ? 6 : 4, index);
        if (ib <= 0) return -1;
        uint32_t used = (uint32_t)ib;
        if (index != 0) {
            if (!hp_copy_indexed(h, index, false, rec, cap, nl, vl, ovf)) return ovf ? -2 : -1;
        } else {
            const int nb = hp_str(p + used, left - used, rec, cap, nl);
            if (nb <= 0) return nb == -2 ? -2 : -1;
            used += (uint32_t)nb;
            for (uint32_t i = 0; i < nl; i++) if (rec[i] >= 'A' && rec[i] <= 'Z') rec[i] = (uint8_t)(rec[i] + 32);
        }
        const int vb = hp_str(p + used, left - used, rec + nl, cap - nl, vl);
        if (vb <= 0) return vb == -2 ? -2 : -1;
        used += (uint32_t)vb;
        if (incremental && hp_add(h, rec, nl, vl) != 0) return -1;
        p += used;
    }
    adv = (uint32_t)(p - p0);
    return 1;
}
// One header block, the way ConsumeHeaders loops HPacker::Decode.  Records: u16 name_len, u16 value_len, name, value.
// status: 0 consumed, 1 ran out of bytes inside a field, -1 malformed, -2 output capacity exceeded
__device__ __noinline__ int hpack_decode_block(HpackState& h, const uint8_t* in, uint32_t n, uint8_t* out, uint32_t out_cap,
                                               uint32_t& out_len, uint32_t& n_headers) {
    uint32_t pos = 0, o = 0, cnt = 0;
    int status = 0;
    while (pos < n) {
        if (o + 4 > out_cap) { status = -2; break; }
        uint32_t nl = 0, vl = 0, adv = 0;
        const int rc = hpack_decode_field(h, in + pos, n - pos, out + o + 4, out_cap - o - 4, nl, vl, adv);
        if (rc <= 0) { status = rc == 0 ? 1 : rc; break; }
        out[o] = (uint8_t)nl; out[o + 1] = (uint8_t)(nl >> 8); out[o + 2] = (uint8_t)vl; out[o + 3] = (uint8_t)(vl >> 8);
        o += 4 + nl + vl; cnt++;
        pos += adv;
    }
    out_len = o; n_headers = cnt;
    return status;
}

struct H2Frame { uint8_t type, flags; uint16_t pad; uint32_t stream_id, payload_off, payload_len; };   // == b2_h2_frame

// blocks [first[g], first[g+1]) belong to one connection and are decoded in order by one thread
__global__ void k_hpack_decode(const uint8_t* bytes, const uint32_t* blk_conn, const uint32_t* blk_off, const uint32_t* blk_len,
                               const uint32_t* group_first, uint32_t n_groups, HpackState* states, uint8_t* out, uint32_t per_block_cap,
                               uint32_t* out_lens, int32_t* status, uint32_t* n_headers) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    for (uint32_t b = group_first[g]; b < group_first[g + 1]; b++) {
        uint32_t ol = 0, nh = 0;
        const int st = hpack_decode_block(states[blk_conn[b]], bytes + blk_off[b], blk_len[b], out + (size_t)b * per_block_cap, per_block_cap, ol, nh);
        out_lens[b] = ol; status[b] = st; n_headers[b] = nh;
    }
}
__global__ void k_hpack_reset(HpackState* states, uint32_t conn, uint32_t max_size) {
    HpackState& h = states[conn];
    h.max_size = max_size; h.size = 0; h.count = 0; h.head = 0; h.byte_head = 0;
}

// one thread per connection run: the chain of 9-byte frame heads
__global__ void k_h2_scan(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, uint32_t max_frame_size, H2Frame* frames,
                          uint32_t cap_per_run, uint32_t* n_frames, uint32_t* consumed, uint32_t* err) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_runs) return;
    const uint8_t* in = bytes + runs[r].offset; const uint32_t n = runs[r].length;
    uint32_t pos = 0, cnt = 0, e = B2_PARSE_ERROR_NOT_ENOUGH_DATA;
    if (runs[r].flags & 2u) {                               // server side, connection start: the 24-byte client preface
        const char* pre = "PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n";
        const uint32_t k = n < 24 ? n : 24;
        bool match = true;
        for (uint32_t i = 0; i < k; i++) if (in[i] != (uint8_t)pre[i]) { match = false; break; }
        if (!match) { n_frames[r] = 0; consumed[r] = 0; err[r] = B2_PARSE_ERROR_TRY_OTHERS; return; }
        if (n < 24) { n_frames[r] = 0; consumed[r] = 0; err[r] = B2_PARSE_ERROR_NOT_ENOUGH_DATA; return; }
        pos = 24;
    }
    H2Frame* out = frames + (size_t)r * cap_per_run;
    for (;;) {
        if (n - pos < 3) break;
        const uint32_t length = ((uint32_t)in[pos] << 16) | ((uint32_t)in[pos + 1] << 8) | in[pos + 2];
        if (length > max_frame_size) { e = B2_PARSE_ERROR_ABSOLUTELY_WRONG; break; }
        if ((unsigned long long)(n - pos - 3) < 6ull + length) break;
        const uint32_t sid = load_be32(in + pos + 5);
        if (sid & 0x80000000u) { e = B2_PARSE_ERROR_ABSOLUTELY_WRONG; break; }
        if (cnt < cap_per_run) {
            H2Frame f; f.type = in[pos + 3]; f.flags = in[pos + 4]; f.pad = 0; f.stream_id = sid;
            f.payload_off = runs[r].offset + pos + 9; f.payload_len = length;
            out[cnt] = f;
        }
        cnt++; pos += 9 + length;
    }
    n_frames[r] = cnt; consumed[r] = pos; err[r] = e;
}

// ---------------------------------------------------------------------------------------------------------
// ParseH2Message: one thread per connection run walks H2Context::Consume (policy/http2_rpc_protocol.cpp:467-543) frame
// by frame.  A connection is a serial state machine (HPACK table, settings, windows, pending streams), so connections
// are the unit of parallelism, exactly like the reference runs one input bthread per socket.  Every quirk of the
// reference that shapes the byte stream is kept: handlers that fail (or PING acks) leave the rest of their payload
// unread and the next "frame head" is parsed from there.  The helpers of both sides and the server's message builder
// are here; the frame loop (h2_consume_run) follows the client's helpers further down.
constexpr uint32_t kH2HdrBytes = B2_H2_HEADER_BYTES;
constexpr long long kH2MaxWindow = 2147483647ll;                 // H2Settings::MAX_WINDOW_SIZE
// n bytes src -> dst by ONE thread: 16-byte words when the pointers agree mod 16, else 4-byte words assembled from
// aligned loads (a connection is a serial state machine; its bulk copies are the only place worth widening)
__device__ __forceinline__ void thread_copy(uint8_t* dst, const uint8_t* src, uint32_t n) {
    uint32_t i = 0;
    if ((((uintptr_t)dst ^ (uintptr_t)src) & 15u) == 0) {
        while (i < n && ((uintptr_t)(dst + i) & 15u)) { dst[i] = src[i]; i++; }
        for (; i + 64 <= n; i += 64) {
            const uint4 a = *reinterpret_cast<const uint4*>(src + i), b = *reinterpret_cast<const uint4*>(src + i + 16);
            const uint4 c = *reinterpret_cast<const uint4*>(src + i + 32), d = *reinterpret_cast<const uint4*>(src + i + 48);
            *reinterpret_cast<uint4*>(dst + i) = a; *reinterpret_cast<uint4*>(dst + i + 16) = b;
            *reinterpret_cast<uint4*>(dst + i + 32) = c; *reinterpret_cast<uint4*>(dst + i + 48) = d;
        }
        for (; i + 16 <= n; i += 16) *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(src + i);
    } else {
        while (i < n && ((uintptr_t)(dst + i) & 3u)) { dst[i] = src[i]; i++; }
        const uint32_t sh = 8u * (uint32_t)((uintptr_t)(src + i) & 3u);
        if (i + 8 <= n) {
            const uint32_t* q = reinterpret_cast<const uint32_t*>((uintptr_t)(src + i) & ~(uintptr_t)3);
            uint32_t w0 = q[0];
            for (; i + 8 <= n; i += 4) {                         // (+8: the look-ahead word stays inside the source)
                const uint32_t w1 = *++q;
                *reinterpret_cast<uint32_t*>(dst + i) = sh ? __funnelshift_r(w0, w1, sh) : w0;
                w0 = w1;
            }
        }
    }
    for (; i < n; i++) dst[i] = src[i];
}
struct H2Stream {
    int32_t id; uint32_t hdr_len, n_headers, body_len;
    uint32_t stream_ended, body_input_off;                       // body_input_off: the whole body is one DATA payload of THIS batch (0 = it lives in the slot)
    long long remote_window_left, deferred_wu;
};
struct H2Conn {
    uint32_t conn_state; int32_t last_received_stream_id; uint32_t remote_settings_received, n_pending;
    uint32_t r_header_table_size, r_enable_push, r_max_concurrent_streams, r_stream_window_size, r_max_frame_size, r_max_header_list_size;
    uint32_t l_stream_window_size, l_max_frame_size;
    long long remote_window_left, deferred_window_update;
    long long last_sent_stream_id; uint32_t preface_sent, pad0;  // client side: H2Context::_last_sent_stream_id (:331); the preface goes out with the first request
    HpackState enc;                                              // HPacker::_encode_table (responses)
};
// Pending streams live outside H2Conn so that their number and size are run-time choices (b2_h2_configure): connection i
// owns streams[i * pending ...] and slots[(i * pending + k) * stream_bytes ...]: [0, kH2HdrBytes) header records, then the body.
struct H2Pool { H2Stream* streams; uint8_t* slots; uint32_t pending, stream_bytes; };
struct H2Out {                      // this run's slice of the output buffer
    uint8_t* base; uint32_t ctrl_cap, ctrl_len, blob_off, blob_end; bool overflow;
};
__device__ __forceinline__ void h2_conn_init(H2Conn& c, H2Stream* S, uint32_t P) {
    c.conn_state = 0; c.last_received_stream_id = -1; c.remote_settings_received = 0; c.n_pending = 0;
    // _remote_settings: H2Settings() with the windows maximised (H2Context ctor, :323-345)
    c.r_header_table_size = 4096; c.r_enable_push = 0; c.r_max_concurrent_streams = 0xffffffffu;
    c.r_stream_window_size = (uint32_t)kH2MaxWindow; c.r_max_frame_size = 16384; c.r_max_header_list_size = 0xffffffffu;
    c.l_stream_window_size = 256 * 1024; c.l_max_frame_size = 16384;     // H2Settings() defaults, http2.cpp:26-34
    c.remote_window_left = kH2MaxWindow; c.deferred_window_update = 0;
    c.last_sent_stream_id = 1; c.preface_sent = 0; c.pad0 = 0;
    for (uint32_t i = 0; i < P; i++) S[i].id = -1;
    c.enc.max_size = 4096; c.enc.size = 0; c.enc.count = 0; c.enc.head = 0; c.enc.byte_head = 0;   // _hpacker.Init(header_table_size), :367
}
__device__ __forceinline__ void h2_put_head(uint8_t* p, uint32_t payload, uint8_t type, uint8_t flags, uint32_t sid) {   // SerializeFrameHead :123-136
    p[0] = (uint8_t)(payload >> 16); p[1] = (uint8_t)(payload >> 8); p[2] = (uint8_t)payload; p[3] = type; p[4] = flags;
    p[5] = (uint8_t)(sid >> 24); p[6] = (uint8_t)(sid >> 16); p[7] = (uint8_t)(sid >> 8); p[8] = (uint8_t)sid;
}
__device__ __forceinline__ uint8_t* h2_ack_room(H2Out& o, uint32_t n) {                  // WriteAck :144-150
    if (o.ctrl_len + n > o.ctrl_cap) { o.overflow = true; return nullptr; }
    uint8_t* p = o.base + o.ctrl_len; o.ctrl_len += n; return p;
}
__device__ __forceinline__ void h2_write_wu(H2Out& o, uint32_t sid, long long inc) {
    uint8_t* p = h2_ack_room(o, 13); if (!p) return;
    h2_put_head(p, 4, 8, 0, sid); put_be32(p + 9, (uint32_t)inc);
}
// AddWindowSize (:261-281), literally: the sum is stored even when the check fails
__device__ __forceinline__ bool h2_add_window(long long& w, long long diff) {
    const long long before = w; w = before + diff;
    const long long mask = (long long)(int)0x80000000;            // `(1 << 31)` promoted to int64
    if ((((before | diff) >> 31) & 1) == 0) { if ((before + diff) & mask) return false; }
    if ((((before & diff) >> 31) & 1) == 1) { if (((before + diff) & mask) == 0) return false; }
    return true;
}
__device__ __forceinline__ void h2_defer_wu(H2Conn& c, H2Out& o, long long size) {         // H2Context::DeferWindowUpdate :1078-1094
    if (size <= 0) return;
    c.deferred_window_update += size;
    if (c.deferred_window_update >= (long long)(c.l_stream_window_size / 2)) {
        const long long conn_wu = c.deferred_window_update; c.deferred_window_update = 0;
        if (conn_wu > 0) h2_write_wu(o, 0, conn_wu);
    }
}
// the flow control of H2StreamContext::OnData (:743-774) on a stream's deferred WINDOW_UPDATE; false = FLOW_CONTROL_ERROR
__device__ __forceinline__ bool h2_data_quota(H2Conn& c, H2Out& o, int32_t sid, long long& deferred, uint32_t frag) {
    const long long acc = (long long)frag + deferred; deferred += frag;
    const long long quota = (long long)(c.l_stream_window_size / (c.n_pending + 1));
    if (acc >= quota) {
        if (acc > (long long)c.l_stream_window_size) return false;
        const long long swu = deferred; deferred = 0;
        if (swu > 0) { h2_write_wu(o, (uint32_t)sid, swu); const long long cw = swu + c.deferred_window_update; c.deferred_window_update = 0; h2_write_wu(o, 0, cw); }
    }
    return true;
}
__device__ __forceinline__ int h2_find(const H2Stream* S, uint32_t P, int32_t id) {
    for (uint32_t i = 0; i < P; i++) if (S[i].id == id) return (int)i;
    return -1;
}
// RemoveStreamAndDeferWU (:378-392); returns the slot (the caller still reads the stream's data) or -1
__device__ __forceinline__ int h2_remove_stream(H2Conn& c, H2Stream* S, uint32_t P, H2Out& o, int32_t id) {
    const int k = h2_find(S, P, id);
    if (k < 0) return -1;
    S[k].id = -1; c.n_pending--;
    const long long d = S[k].deferred_wu; S[k].deferred_wu = 0;
    h2_defer_wu(c, o, d);
    return k;
}
__device__ __forceinline__ bool ci_eq(const uint8_t* a, uint32_t n, const char* lit) {    // strcasecmp(a (c_str of n bytes), lit) == 0
    uint32_t i = 0;
    for (; lit[i]; i++) {
        if (i >= n) return false;
        uint8_t x = a[i]; if (x >= 'a' && x <= 'z') x = (uint8_t)(x - 32);
        if (x != (uint8_t)lit[i]) return false;
    }
    return i == n;
}
__device__ __forceinline__ uint32_t cstr_len(const uint8_t* p, uint32_t n) {           // strnlen: four bytes per step
    uint32_t i = 0;
    for (; i + 4 <= n; i += 4) {
        const uint32_t z = __vcmpeq4(ld32_any(p + i), 0u);
        if (z) return i + ((__ffs(z) - 1) >> 3);
    }
    while (i < n && p[i]) i++;
    return i;
}
__device__ __forceinline__ bool lit_eq(const uint8_t* a, uint32_t n, const char* lit) {   // strcmp(c_str, lit) == 0
    uint32_t i = 0;
    for (; lit[i]; i++) if (i >= n || a[i] != (uint8_t)lit[i]) return false;
    return i == n;
}
__device__ __forceinline__ bool has_prefix(const uint8_t* a, uint32_t n, const char* lit, uint32_t& l) {
    l = 0; while (lit[l]) { if (l >= n || a[l] != (uint8_t)lit[l]) return false; l++; }
    return true;
}
// Str2HttpMethod (http_method.cpp:104-140): case-insensitive exact match of the c_str against the 27 names
__device__ __forceinline__ int h2_http_method(const uint8_t* v, uint32_t vl) {
    const uint32_t n = cstr_len(v, vl);
    const char* const names[27] = { "DELETE", "GET", "HEAD", "POST", "PUT", "CONNECT", "OPTIONS", "TRACE", "COPY", "LOCK", "MKCOL", "MOVE",
        "PROPFIND", "PROPPATCH", "SEARCH", "UNLOCK", "REPORT", "MKACTIVITY", "CHECKOUT", "MERGE", "M-SEARCH", "NOTIFY", "SUBSCRIBE",
        "UNSUBSCRIBE", "PATCH", "PURGE", "MKCALENDAR" };
    for (int m = 0; m < 27; m++) if (ci_eq(v, n, names[m])) return m;
    return -1;
}
// ParseContentType (policy/http_rpc_protocol.cpp:176-230)
__device__ __forceinline__ uint32_t h2_content_type(const uint8_t* ct, uint32_t n, bool& is_grpc) {
    is_grpc = false;
    uint32_t l;
    if (!has_prefix(ct, n, "application/", l)) return 0;
    ct += l; n -= l;
    if (has_prefix(ct, n, "grpc", l)) {
        if (n == 4 || ct[4] == ';') { is_grpc = true; return 2; }
        else if (ct[4] == '+') { ct += 5; n -= 5; is_grpc = true; }
    }
    uint32_t type;
    if (has_prefix(ct, n, "json", l)) type = 1;
    else if (has_prefix(ct, n, "proto-json", l)) type = 4;
    else if (has_prefix(ct, n, "proto-text", l)) type = 3;
    else if (has_prefix(ct, n, "proto", l)) type = 2;
    else if (has_prefix(ct, n, "x-protobuf", l)) type = 2;
    else return 0;
    ct += l; n -= l;
    return (n == 0 || ct[0] == ';') ? type : 0;
}
// one header of ConsumeHeaders (:1232-1287): false = the reference returns -1
__device__ __forceinline__ bool h2_check_header(const uint8_t* name, uint32_t nl, const uint8_t* value, uint32_t vl) {
    const uint32_t n = cstr_len(name, nl);
    if (n == 0 || name[0] != ':') return true;
    const uint8_t c1 = n > 1 ? name[1] : 0;
    const uint8_t* rest = name + 2; const uint32_t rn = n > 2 ? n - 2 : 0;
    switch (c1) {
    case 'a': return lit_eq(rest, rn, "uthority");
    case 'm': return lit_eq(rest, rn, "ethod") && h2_http_method(value, vl) >= 0;
    case 'p': return lit_eq(rest, rn, "ath");
    case 's':
        if (lit_eq(rest, rn, "cheme")) return true;
        if (lit_eq(rest, rn, "tatus")) {                 // strtol(value, &end, 10) must stop at the terminating NUL
            const uint32_t m = cstr_len(value, vl);
            uint32_t i = 0;
            while (i < m && (value[i] == ' ' || (value[i] >= 9 && value[i] <= 13))) i++;
            uint32_t j = i;
            if (j < m && (value[j] == '+' || value[j] == '-')) j++;
            uint32_t d = j; while (d < m && value[d] >= '0' && value[d] <= '9') d++;
            const uint32_t end = d > j ? d : 0;          // no digits: endptr = nptr
            return end == m;
        }
        return false;
    default: return false;
    }
}
struct H2Res { int kind; uint32_t err; int32_t err_stream; int slot; };   // kind 0 ok, 1 ok + message in `slot`, 2 error
__device__ __forceinline__ H2Res h2_ok() { H2Res r; r.kind = 0; r.err = 0; r.err_stream = 0; r.slot = -1; return r; }
__device__ __forceinline__ H2Res h2_err(uint32_t e, int32_t sid = 0) { H2Res r; r.kind = 2; r.err = e; r.err_stream = sid; r.slot = -1; return r; }

// H2StreamContext::ConsumeHeaders over one fragment, records appended to the stream's slot
__device__ __forceinline__ int h2_consume_headers(H2Conn& c, HpackState& hp, H2Stream& st, uint8_t* slot, const uint8_t* frag, uint32_t n, bool& no_room) {
    uint32_t pos = 0;
    while (pos < n) {
        if (st.hdr_len + 4 > kH2HdrBytes) { no_room = true; return -1; }
        uint8_t* rec = slot + st.hdr_len;
        uint32_t nl = 0, vl = 0, adv = 0;
        const int rc = hpack_decode_field(hp, frag + pos, n - pos, rec + 4, kH2HdrBytes - st.hdr_len - 4, nl, vl, adv);
        if (rc == -2) { no_room = true; return -1; }
        if (rc < 0) return -1;
        if (rc == 0) break;
        if (!h2_check_header(rec + 4, nl, rec + 4 + nl, vl)) return -1;
        rec[0] = (uint8_t)nl; rec[1] = (uint8_t)(nl >> 8); rec[2] = (uint8_t)vl; rec[3] = (uint8_t)(vl >> 8);
        st.hdr_len += 4 + nl + vl; st.n_headers++;
        pos += adv;
    }
    return 0;
}
// OnEndStream (:823-846): the stream leaves the pending map; the caller emits the message from its slot
__device__ __forceinline__ H2Res h2_end_stream(H2Conn& c, H2Stream* S, uint32_t P, H2Out& o, int32_t id) {
    const int k = h2_remove_stream(c, S, P, o, id);
    if (k < 0) return h2_ok();
    H2Res r = h2_ok(); r.kind = 1; r.slot = k; r.err_stream = id; return r;
}

__global__ void k_h2_conn_reset(H2Conn* conns, HpackState* hps, uint32_t conn, H2Pool pool) {
    h2_conn_init(conns[conn], pool.streams + (size_t)conn * pool.pending, pool.pending);
    HpackState& h = hps[conn]; h.max_size = 4096; h.size = 0; h.count = 0; h.head = 0; h.byte_head = 0;
}

// RemoveGrpcPrefix (policy/http_rpc_protocol.cpp:264-277) of a body that sits at `body_off` in the descriptors' offsets
struct H2GrpcMsg { bool prefix_ok, compressed; uint32_t msg_off, msg_len; };
__device__ __forceinline__ H2GrpcMsg h2_remove_grpc_prefix(const uint8_t* body, uint32_t body_len, uint32_t body_off) {
    H2GrpcMsg g; g.prefix_ok = false; g.compressed = false; g.msg_off = 0; g.msg_len = 0;
    if (body_len == 0) { g.prefix_ok = true; g.msg_off = body_off; }
    else if (body_len >= 5) {
        g.compressed = body[0] != 0;
        if ((unsigned long long)load_be32(body + 1) + 5ull == body_len) { g.prefix_ok = true; g.msg_off = body_off + 5; g.msg_len = body_len - 5; }
    }
    return g;
}
// The completed request on a server connection, as ProcessHttpRequest first sees it: the stream (already out of the pending map; its
// bytes are still in `slot`) becomes one b2_h2_msg.  False when the run's descriptors or blob space ran out.
__device__ __forceinline__ bool h2_emit_msg(const H2Stream& st, const uint8_t* slot, int32_t sid, uint32_t r, uint32_t gbase, H2Out& o, const uint8_t* bytes,
                                            const DevMethod* methods, uint32_t n_methods, b2_h2_msg* mout, uint32_t& n_msgs, uint32_t cap) {
    const bool in_input = st.body_input_off != 0;
    const uint32_t need = ((st.hdr_len + 15u) & ~15u) + (in_input ? 0u : ((st.body_len + 15u) & ~15u));
    if (n_msgs >= cap || o.blob_off + need > o.blob_end) return false;
    b2_h2_msg m;
    m.run_idx = r; m.stream_id = (uint32_t)sid; m.reserved = 0;
    const uint32_t ho = o.blob_off, bo = ho + ((st.hdr_len + 15u) & ~15u);
    thread_copy(o.base + ho, slot, st.hdr_len);
    if (!in_input) thread_copy(o.base + bo, slot + kH2HdrBytes, st.body_len);
    o.blob_off += need;
    m.headers_off = gbase + ho; m.headers_len = st.hdr_len; m.n_headers = st.n_headers;
    m.body_off = in_input ? st.body_input_off : gbase + bo; m.body_len = st.body_len;
    m.http_method = B2_H2_NO_METHOD; m.content_type = 0; m.flags = 0; m.method_idx = -1;
    m.msg_off = 0; m.msg_len = 0; m.path_off = 0; m.path_len = 0;
    if (in_input) m.flags |= B2_H2_FLAG_BODY_IN_INPUT;
    const uint8_t* body_p = in_input ? bytes + st.body_input_off : slot + kH2HdrBytes;
    bool is_grpc = false;
    const uint8_t* path = nullptr; uint32_t path_len = 0;
    for (uint32_t q = 0; q < st.hdr_len;) {
        const uint32_t nl = slot[q] | ((uint32_t)slot[q + 1] << 8), vl = slot[q + 2] | ((uint32_t)slot[q + 3] << 8);
        const uint8_t* nm = slot + q + 4; const uint8_t* v = nm + nl;
        const uint32_t cn = cstr_len(nm, nl);
        if (lit_eq(nm, cn, ":method")) m.http_method = (uint32_t)h2_http_method(v, vl);
        else if (lit_eq(nm, cn, ":path")) {                  // URI::SetH2Path (uri.cpp:403-425): up to '?' / '#'
            uint32_t e = 0; while (e < vl && v[e] && v[e] != '?' && v[e] != '#') e++;
            path = v; path_len = e; m.path_off = gbase + ho + (uint32_t)(v - slot); m.path_len = e; m.flags |= B2_H2_FLAG_HAS_PATH;
        } else if (lit_eq(nm, cn, "content-type")) m.content_type = h2_content_type(v, vl, is_grpc);
        q += 4 + nl + vl;
    }
    if (is_grpc) {
        m.flags |= B2_H2_FLAG_GRPC;
        const H2GrpcMsg g = h2_remove_grpc_prefix(body_p, st.body_len, m.body_off);
        if (g.prefix_ok) m.flags |= B2_H2_FLAG_GRPC_PREFIX_OK;
        if (g.compressed) m.flags |= B2_H2_FLAG_GRPC_COMPRESSED;
        m.msg_off = g.msg_off; m.msg_len = g.msg_len;
    }
    if (path) {
        // FindMethodPropertyByURIImpl (:1088-1138), "[service]/[method]" form: '/'-separated, empty fields skipped
        uint32_t f0 = 0; while (f0 < path_len && path[f0] == '/') f0++;
        uint32_t e0 = f0; while (e0 < path_len && path[e0] != '/') e0++;
        uint32_t f1 = e0; while (f1 < path_len && path[f1] == '/') f1++;
        uint32_t e1 = f1; while (e1 < path_len && path[e1] != '/') e1++;
        if (e0 > f0 && e1 > f1) {
            bool no_service = false;
            m.method_idx = find_method(methods, n_methods, path + f0, e0 - f0, path + f1, e1 - f1, no_service);
        }
    }
    mout[n_msgs++] = m;
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// Response side: H2UnsentResponse::AppendAndDestroySelf (:1688-1750) + PackH2Message (:1310-1380), one thread per connection.
__device__ __forceinline__ uint8_t lc(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }
__device__ __forceinline__ uint8_t* hp_put_int(uint8_t* p, uint8_t msb, uint32_t prefix, uint32_t value) {       // EncodeInteger :479-496
    const uint32_t lim = (1u << prefix) - 1;
    if (value < lim) { *p++ = (uint8_t)(msb | value); return p; }
    value -= lim; *p++ = (uint8_t)(msb | lim);
    for (; value >= 128;) { *p++ = (uint8_t)((value & 0x7f) | 0x80); value >>= 7; }
    *p++ = (uint8_t)value;
    return p;
}
// the encoder's view of "is this header / this name in a table": static first, then the connection's encode table;
// names compare case-insensitively, entries with an empty value are never full matches (IndexTable::AddHeader :165-171)
__device__ __forceinline__ uint32_t hp_enc_find(const HpackState& t, const uint8_t* n, uint32_t nl, const uint8_t* v, uint32_t vl, bool want_value) {
    for (uint32_t i = 0; i < 61; i++) {                          // reverse insertion => the smallest index wins for names
        if (kHpackStaticName[i][1] != nl) continue;
        if (want_value && (vl == 0 || kHpackStaticValue[i][1] != vl)) continue;
        bool eq = true;
        for (uint32_t k = 0; k < nl && eq; k++) eq = lc(n[k]) == lc(kHpackStaticBlob[kHpackStaticName[i][0] + k]);
        for (uint32_t k = 0; want_value && k < vl && eq; k++) eq = v[k] == kHpackStaticBlob[kHpackStaticValue[i][0] + k];
        if (eq) return i + 1;
    }
    for (uint32_t i = 0; i < t.count; i++) {                     // newest first == the latest id of a duplicated header
        const uint32_t e = (t.head + i) & 127u;
        if (t.meta[e].nl != nl) continue;
        if (want_value && (vl == 0 || t.meta[e].vl != vl)) continue;
        bool eq = true;
        for (uint32_t k = 0; k < nl && eq; k++) eq = lc(n[k]) == lc(t.bytes[(t.meta[e].off + k) & 4095u]);
        for (uint32_t k = 0; want_value && k < vl && eq; k++) eq = v[k] == t.bytes[(t.meta[e].off + nl + k) & 4095u];
        if (eq) return 62 + i;
    }
    return 0;
}
// HPacker::Encode (:696-726); hp_add wants name||value contiguous: `tmp` (>= nl + vl bytes) is scratch
__device__ __forceinline__ uint8_t* hp_encode(HpackState& t, uint8_t* p, const uint8_t* n, uint32_t nl, const uint8_t* v, uint32_t vl, bool never_index, uint8_t* tmp) {
    if (!never_index) {
        const uint32_t idx = hp_enc_find(t, n, nl, v, vl, true);
        if (idx) return hp_put_int(p, 0x80, 7, idx);
    }
    const uint32_t name_index = hp_enc_find(t, n, nl, nullptr, 0, false);
    if (!never_index) {
        for (uint32_t k = 0; k < nl; k++) tmp[k] = n[k];
        for (uint32_t k = 0; k < vl; k++) tmp[nl + k] = v[k];
        (void)hp_add(t, tmp, nl, vl);
        p = hp_put_int(p, 0x40, 6, name_index);
    } else p = hp_put_int(p, 0x10, 4, name_index);
    if (name_index == 0) { p = hp_put_int(p, 0x00, 7, nl); for (uint32_t k = 0; k < nl; k++) *p++ = lc(n[k]); }
    p = hp_put_int(p, 0x00, 7, vl); for (uint32_t k = 0; k < vl; k++) *p++ = v[k];
    return p;
}
__device__ __forceinline__ uint32_t put_dec_i32_h2(uint8_t* p, int32_t v) {     // "%d"
    uint8_t tmp[12]; uint32_t n = 0; uint32_t u = v < 0 ? (uint32_t)(-(long long)v) : (uint32_t)v;
    do { tmp[n++] = (uint8_t)('0' + u % 10); u /= 10; } while (u);
    uint32_t o = 0; if (v < 0) p[o++] = '-';
    while (n) p[o++] = tmp[--n];
    return o;
}
constexpr uint32_t kH2FragCap = 1024;      // encoded header block of one response (":status", "content-type", trailers)
constexpr uint32_t kH2PackWarps = 4;
// The out bytes one reply of k_h2_pack may take, reserved by b2_h2_pack_responses and b2_h2_serve_batch alike: DATA (the body + the
// 5-byte gRPC prefix) with a frame head per max_frame_size (>= 16384) piece, HEADERS + trailers (each header at most twice its bytes
// + 64 once encoded), the deferred WINDOW_UPDATE and 16 bytes of slack.
B2_HD uint64_t h2_reply_bound(uint32_t body_len, uint32_t content_type_len, uint32_t grpc_message_len) {
    const uint64_t data = (uint64_t)body_len + 5;
    return data + 9 * (data / 16384 + 4) + 2ull * (content_type_len + grpc_message_len + 64) + 13 + 16;
}
// One WARP per connection: lane 0 runs the serial part (window check, HPACK encode against the connection's table,
// deferred WINDOW_UPDATE) into shared memory, then the whole warp writes the frames — the DATA payload, which is
// nearly all of the bytes, with coalesced 16-byte copies.
// Connection group g, by one warp; buf: the warp's 3 * kH2FragCap bytes of shared scratch.  k_h2_pack and k_h2_ring call it.
__device__ __forceinline__ void h2_pack_group(uint32_t g, uint32_t lane, uint8_t* buf, const uint8_t* bytes, const uint8_t* last_input, const uint8_t* last_out,
                                              const b2_h2_response* resps, const uint32_t* group_first, H2Conn* conns,
                                              uint8_t* out, const uint32_t* out_offs, uint32_t* out_lens) {
    uint8_t* frag = buf; uint8_t* trailer = buf + kH2FragCap; uint8_t* tmp = buf + 2 * kH2FragCap;
    for (uint32_t i = group_first[g]; i < group_first[g + 1]; i++) {
        const b2_h2_response R = resps[i];
        uint8_t* o0 = out + out_offs[i]; uint8_t* o = o0;
        const bool grpc = R.flags & B2_H2_RESP_GRPC;
        const uint32_t data_size = R.body_len + (grpc ? 5u : 0u);
        uint32_t rst = 0, fl = 0, tl = 0, mfs = 0, cw = 0;
        if (lane == 0) {
            H2Conn& c = conns[R.conn];
            // MinusWindowSize(&_remote_window_left, _data.size()) (:283-296)
            if (c.remote_window_left < (long long)data_size) rst = 1;
            else {
                c.remote_window_left -= (long long)data_size;
                const bool never = c.r_header_table_size == 0;
                uint8_t num[16];
                uint8_t* f = frag;
                { const uint32_t nn = put_dec_i32_h2(num, R.status_code); f = hp_encode(c.enc, f, (const uint8_t*)":status", 7, num, nn, never, tmp); }
                if (R.content_type_len) f = hp_encode(c.enc, f, (const uint8_t*)"content-type", 12, ((R.flags & B2_H2_RESP_CT_IN_OUT) ? last_out : bytes) + R.content_type_off, R.content_type_len, never, tmp);
                uint8_t* t = trailer;
                if (grpc) {
                    const uint32_t nn = put_dec_i32_h2(num, R.grpc_status);
                    t = hp_encode(c.enc, t, (const uint8_t*)"grpc-status", 11, num, nn, never, tmp);
                    if (R.grpc_message_len) t = hp_encode(c.enc, t, (const uint8_t*)"grpc-message", 12, bytes + R.grpc_message_off, R.grpc_message_len, never, tmp);
                }
                fl = (uint32_t)(f - frag); tl = (uint32_t)(t - trailer); mfs = c.r_max_frame_size;
                if (c.deferred_window_update > 0) { cw = (uint32_t)c.deferred_window_update; c.deferred_window_update = 0; }   // ReleaseDeferredWindowUpdate
            }
        }
        rst = __shfl_sync(0xffffffffu, rst, 0); fl = __shfl_sync(0xffffffffu, fl, 0); tl = __shfl_sync(0xffffffffu, tl, 0);
        mfs = __shfl_sync(0xffffffffu, mfs, 0); cw = __shfl_sync(0xffffffffu, cw, 0);
        __syncwarp();
        if (rst) {                                                   // RST_STREAM(FLOW_CONTROL_ERROR) instead of the response (:1706-1712)
            if (lane == 0) { h2_put_head(o, 4, 3, 0, R.stream_id); put_be32(o + 9, 3); out_lens[i] = 13; }
            __syncwarp();
            continue;
        }
        // ---- PackH2Message (:1310-1380)
        const uint8_t hflags = (data_size == 0 && tl == 0) ? 0x1 : 0;
        if (fl <= mfs) {
            if (lane == 0) h2_put_head(o, fl, 1, hflags | 0x4, R.stream_id);
            for (uint32_t k = lane; k < fl; k += 32) o[9 + k] = frag[k];
            o += 9 + fl;
        } else {                                                     // (cannot happen with kH2FragCap < 16384 <= max_frame_size; kept for the shape)
            if (lane == 0) {
                uint8_t* q = o;
                h2_put_head(q, mfs, 1, hflags, R.stream_id); q += 9; for (uint32_t k = 0; k < mfs; k++) *q++ = frag[k];
                for (uint32_t at = mfs; at < fl;) { const uint32_t nn = min(fl - at, mfs); h2_put_head(q, nn, 9, at + nn == fl ? 0x4 : 0, R.stream_id); q += 9; for (uint32_t k = 0; k < nn; k++) *q++ = frag[at + k]; at += nn; }
            }
            o += fl + 9 * ((fl + mfs - 1) / mfs);
        }
        const uint8_t* body = ((R.flags & B2_H2_RESP_BODY_IN_INPUT) ? last_input : (R.flags & B2_H2_RESP_BODY_IN_OUT) ? last_out : bytes) + R.body_off;
        for (uint32_t at = 0; at < data_size;) {
            const uint32_t nn = min(data_size - at, mfs);
            const uint8_t dflags = (at + nn == data_size && tl == 0) ? 0x1 : 0;
            if (lane == 0) h2_put_head(o, nn, 0, dflags, R.stream_id);
            o += 9;
            uint32_t k = 0;
            if (grpc && at < 5) { k = min(nn, 5u - at); if (lane < k) { const uint32_t q = at + lane; o[lane] = q == 0 ? 0 : (uint8_t)(R.body_len >> (8 * (4 - q))); } }   // AddGrpcPrefix: flag 0 + BE32 length
            warp_copy(o + k, body + (at + k - (grpc ? 5u : 0u)), nn - k, lane);
            o += nn; at += nn;
        }
        if (tl) { if (lane == 0) h2_put_head(o, tl, 1, 0x5, R.stream_id); for (uint32_t k = lane; k < tl; k += 32) o[9 + k] = trailer[k]; o += 9 + tl; }
        if (cw) { if (lane == 0) { h2_put_head(o, 4, 8, 0, 0); put_be32(o + 9, cw); } o += 13; }
        if (lane == 0) out_lens[i] = (uint32_t)(o - o0);
        __syncwarp();                                                // the shared buffers are reused by the next response
    }
}
__global__ void __launch_bounds__(kH2PackWarps * 32) k_h2_pack(const uint8_t* bytes, const uint8_t* last_input, const uint8_t* last_out, const b2_h2_response* resps,
                                                               const uint32_t* group_first, uint32_t n_groups, H2Conn* conns,
                                                               uint8_t* out, const uint32_t* out_offs, uint32_t* out_lens) {
    __shared__ __align__(16) uint8_t s_buf[kH2PackWarps][3][kH2FragCap];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * kH2PackWarps + w;
    if (g >= n_groups) return;
    h2_pack_group(g, lane, s_buf[w][0], bytes, last_input, last_out, resps, group_first, conns, out, out_offs, out_lens);
}

// ---------------------------------------------------------------------------------------------------------
constexpr uint32_t kH2ClientMode = 1u;                            // H2Conn::pad0 bit of a connection opened by k_h2_client_conn_reset
// Client side: H2UnsentRequest::New (:1382-1453, the header list) + AppendAndDestroySelf (:1496-1592) + PackH2Message (:1310-1380).
// The same split as k_h2_pack: one warp per connection, lane 0 runs the serial part (stream id, windows, HPACK encode against the
// connection's table) into shared memory, the warp writes the frames.
constexpr uint32_t kH2ReqFragCap = 2048;
// Connection group g, by one warp; buf: the warp's 2 * kH2ReqFragCap bytes of shared scratch; results[i].out_off placed by the host.
// k_h2_pack_req and k_h2_client_ring call it.
__device__ __forceinline__ void h2_pack_req_group(uint32_t g, uint32_t lane, uint8_t* buf, const uint8_t* bytes, const b2_h2_request* reqs,
                                                  const uint32_t* group_first, H2Conn* conns, uint8_t* out, b2_h2_request_result* results, H2Pool pool) {
    uint8_t* frag = buf; uint8_t* tmp = buf + kH2ReqFragCap;
    for (uint32_t i = group_first[g]; i < group_first[g + 1]; i++) {
        const b2_h2_request R = reqs[i];
        uint8_t* o0 = out + results[i].out_off; uint8_t* o = o0;
        const bool grpc = R.flags & B2_H2_REQ_GRPC;
        const uint32_t data_size = R.body_len + (grpc ? 5u : 0u);
        uint32_t st = B2_H2_REQ_OK, sid = 0, fl = 0, mfs = 0, cw = 0, pre = 0;
        if (lane == 0) {
            H2Conn& c = conns[R.conn];
            if (!c.preface_sent) { c.preface_sent = 1; pre = 1; }
            // a connection whose frames the device parses (k_h2_client_conn_reset) also keeps the pending-stream map of
            // AppendAndDestroySelf / TryToInsertStream (:1529-1564, :425-436); the pool slot is a device capacity checked up front
            const bool client = c.pad0 & kH2ClientMode;
            H2Stream* const S = pool.streams + (size_t)R.conn * pool.pending;
            int slot = -1;
            if (client && c.n_pending > c.r_max_concurrent_streams) st = B2_H2_REQ_ELIMIT;                      // no id consumed
            else if (client && (slot = h2_find(S, pool.pending, -1)) < 0) st = B2_H2_REQ_NO_ROOM;
            else if (c.last_sent_stream_id > 0x7FFFFFFFll) st = B2_H2_REQ_RUNOUT;                      // AllocateClientStreamId
            else {
                sid = (uint32_t)c.last_sent_stream_id; c.last_sent_stream_id += 2;
                // ConsumeWindowSize (:1199-1219) on a stream that starts with the peer's initial window (Init :1176-1181)
                if (data_size && ((long long)c.r_stream_window_size < (long long)data_size || c.remote_window_left < (long long)data_size)) st = B2_H2_REQ_ELIMIT;
                else if (client && c.last_received_stream_id >= 0 && (int32_t)sid > c.last_received_stream_id) {   // after GOAWAY (_goaway_stream_id)
                    c.remote_window_left -= (long long)data_size;                  // (taken by ConsumeWindowSize before TryToInsertStream refuses)
                    st = B2_H2_REQ_LOGOFF;
                } else {
                    if (client) {
                        H2Stream& ns = S[slot];
                        ns.id = (int32_t)sid; ns.hdr_len = 0; ns.n_headers = 0; ns.body_len = 0; ns.stream_ended = 0; ns.body_input_off = 0;
                        ns.remote_window_left = (long long)c.r_stream_window_size - (long long)data_size; ns.deferred_wu = 0;
                        c.n_pending++;
                    }
                    c.remote_window_left -= (long long)data_size;
                    const bool never = c.r_header_table_size == 0;
                    uint8_t* f = frag;
                    f = (R.flags & B2_H2_REQ_GET) ? hp_encode(c.enc, f, (const uint8_t*)":method", 7, (const uint8_t*)"GET", 3, never, tmp)
                                                  : hp_encode(c.enc, f, (const uint8_t*)":method", 7, (const uint8_t*)"POST", 4, never, tmp);
                    f = (R.flags & B2_H2_REQ_HTTPS) ? hp_encode(c.enc, f, (const uint8_t*)":scheme", 7, (const uint8_t*)"https", 5, never, tmp)
                                                    : hp_encode(c.enc, f, (const uint8_t*)":scheme", 7, (const uint8_t*)"http", 4, never, tmp);
                    f = hp_encode(c.enc, f, (const uint8_t*)":path", 5, bytes + R.path_off, R.path_len, never, tmp);
                    f = hp_encode(c.enc, f, (const uint8_t*)":authority", 10, bytes + R.authority_off, R.authority_len, never, tmp);
                    if (R.content_type_len) f = hp_encode(c.enc, f, (const uint8_t*)"content-type", 12, bytes + R.content_type_off, R.content_type_len, never, tmp);
                    if (R.flags & B2_H2_REQ_ACCEPT) f = hp_encode(c.enc, f, (const uint8_t*)"accept", 6, (const uint8_t*)"*/*", 3, never, tmp);
                    if (R.flags & B2_H2_REQ_USER_AGENT) f = hp_encode(c.enc, f, (const uint8_t*)"user-agent", 10, (const uint8_t*)"brpc/1.0 curl/7.0", 17, never, tmp);
                    for (uint32_t at = 0; at + 4 <= R.extra_len;) {
                        const uint8_t* e = bytes + R.extra_off + at;
                        const uint32_t nl = e[0] | ((uint32_t)e[1] << 8), vl = e[2] | ((uint32_t)e[3] << 8);
                        if (at + 4 + nl + vl > R.extra_len) break;
                        f = hp_encode(c.enc, f, e + 4, nl, e + 4 + nl, vl, never, tmp);
                        at += 4 + nl + vl;
                    }
                    fl = (uint32_t)(f - frag); mfs = c.r_max_frame_size;
                    if (c.deferred_window_update > 0) { cw = (uint32_t)c.deferred_window_update; c.deferred_window_update = 0; }
                }
            }
        }
        st = __shfl_sync(0xffffffffu, st, 0); sid = __shfl_sync(0xffffffffu, sid, 0); fl = __shfl_sync(0xffffffffu, fl, 0);
        mfs = __shfl_sync(0xffffffffu, mfs, 0); cw = __shfl_sync(0xffffffffu, cw, 0); pre = __shfl_sync(0xffffffffu, pre, 0);
        __syncwarp();
        if (pre) {                                                   // preface + SerializeH2SettingsFrameAndWU(default client settings) (:1508-1526)
            if (lane < 24) o[lane] = (uint8_t)"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n"[lane];
            if (lane == 0) {
                uint8_t* p = o + 24;
                h2_put_head(p, 12, 4, 0, 0);
                p[9] = 0; p[10] = 2; put_be32(p + 11, 0);
                p[15] = 0; p[16] = 4; put_be32(p + 17, 256u * 1024u);
                h2_put_head(p + 21, 4, 8, 0, 0); put_be32(p + 30, 1024u * 1024u - 65535u);
            }
            o += 58;
        }
        if (st != B2_H2_REQ_OK) {
            if (lane == 0) { results[i].status = (int32_t)st; results[i].stream_id = sid; results[i].out_len = (uint32_t)(o - o0); }
            __syncwarp();
            continue;
        }
        const uint8_t hflags = data_size == 0 ? 0x1 : 0;
        if (fl <= mfs) {
            if (lane == 0) h2_put_head(o, fl, 1, hflags | 0x4, sid);
            for (uint32_t k = lane; k < fl; k += 32) o[9 + k] = frag[k];
            o += 9 + fl;
        } else {                                                     // (kH2ReqFragCap < 16384 <= max_frame_size: kept for the shape)
            if (lane == 0) {
                uint8_t* q = o;
                h2_put_head(q, mfs, 1, hflags, sid); q += 9; for (uint32_t k = 0; k < mfs; k++) *q++ = frag[k];
                for (uint32_t at = mfs; at < fl;) { const uint32_t nn = min(fl - at, mfs); h2_put_head(q, nn, 9, at + nn == fl ? 0x4 : 0, sid); q += 9; for (uint32_t k = 0; k < nn; k++) *q++ = frag[at + k]; at += nn; }
            }
            o += fl + 9 * ((fl + mfs - 1) / mfs);
        }
        const uint8_t* body = bytes + R.body_off;
        for (uint32_t at = 0; at < data_size;) {
            const uint32_t nn = min(data_size - at, mfs);
            if (lane == 0) h2_put_head(o, nn, 0, at + nn == data_size ? 0x1 : 0, sid);
            o += 9;
            uint32_t k = 0;
            if (grpc && at < 5) { k = min(nn, 5u - at); if (lane < k) { const uint32_t q = at + lane; o[lane] = q == 0 ? 0 : (uint8_t)(R.body_len >> (8 * (4 - q))); } }   // AddGrpcPrefix
            warp_copy(o + k, body + (at + k - (grpc ? 5u : 0u)), nn - k, lane);
            o += nn; at += nn;
        }
        if (cw) { if (lane == 0) { h2_put_head(o, 4, 8, 0, 0); put_be32(o + 9, cw); } o += 13; }
        if (lane == 0) { results[i].status = B2_H2_REQ_OK; results[i].stream_id = sid; results[i].out_len = (uint32_t)(o - o0); }
        __syncwarp();                                                // the shared buffers are reused by the next request
    }
}
__global__ void __launch_bounds__(kH2PackWarps * 32) k_h2_pack_req(const uint8_t* bytes, const b2_h2_request* reqs, const uint32_t* group_first, uint32_t n_groups,
                                                                   H2Conn* conns, uint8_t* out, b2_h2_request_result* results, H2Pool pool) {
    __shared__ __align__(16) uint8_t s_buf[kH2PackWarps][2][kH2ReqFragCap];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * kH2PackWarps + w;
    if (g >= n_groups) return;
    h2_pack_req_group(g, lane, s_buf[w][0], bytes, reqs, group_first, conns, out, results, pool);
}
// b2_h2_conn_peer_update: OnSettings' effect on _remote_settings (:848-915) and OnWindowUpdate on stream 0 (:1006-1041), mirrored by the host
__global__ void k_h2_peer_update(H2Conn* conns, uint32_t conn, b2_h2_peer_update u, int* rc) {
    H2Conn& c = conns[conn];
    *rc = 0;
    if (u.set & B2_H2_PEER_HEADER_TABLE_SIZE) c.r_header_table_size = u.header_table_size;
    if (u.set & B2_H2_PEER_MAX_FRAME_SIZE) c.r_max_frame_size = u.max_frame_size;
    if (u.set & B2_H2_PEER_STREAM_WINDOW) c.r_stream_window_size = u.stream_window_size;
    if (u.set & B2_H2_PEER_CONN_WINDOW_ADD) {
        if (u.conn_window_add < 0) c.remote_window_left += u.conn_window_add;
        else if (!h2_add_window(c.remote_window_left, u.conn_window_add)) *rc = -1;
    }
}
__global__ void k_h2_set_next_stream_id(H2Conn* conns, uint32_t conn, uint32_t next_id) { conns[conn].last_sent_stream_id = next_id; }

// ---------------------------------------------------------------------------------------------------------
// The receiving half of a client connection: ParseH2Message on a socket created by connect (H2Context::Consume :467-543, client
// branches) -> H2StreamContext::OnEndStream (:825-846) / OnResetStream (:781-823) / OnGoAway (:959-1004) -> what ProcessHttpResponse
// (policy/http_rpc_protocol.cpp:349-564) decides before the response body is parsed.  A connection opened by k_h2_client_conn_reset
// carries kH2ClientMode in H2Conn::pad0; on such a connection H2Conn::last_received_stream_id holds _goaway_stream_id instead (the
// client never updates _last_received_stream_id: it stays -1, which is what its GOAWAY frames carry).  Server connections never
// reach this code, and this code never touches a server connection.
constexpr uint32_t kH2Abandoned = 2u;                             // H2Stream::stream_ended bit on client streams: AddAbandonedStream
constexpr uint32_t kH2ErrMax = 2048;                              // FLAGS_http_max_error_length (http_rpc_protocol.cpp)
__global__ void k_h2_client_conn_reset(H2Conn* conns, HpackState* hps, uint32_t conn, H2Pool pool) {
    // H2Context(socket, NULL) + Init (:324-371): at the default client flags _unack_local_settings equals H2Settings(), which is also
    // _local_settings until the server ACKs, so l_stream_window_size / l_max_frame_size need no second copy
    h2_conn_init(conns[conn], pool.streams + (size_t)conn * pool.pending, pool.pending);
    conns[conn].pad0 = kH2ClientMode;                             // (last_received_stream_id = -1 = _goaway_stream_id)
    HpackState& h = hps[conn]; h.max_size = 4096; h.size = 0; h.count = 0; h.head = 0; h.byte_head = 0;
}
// AddAbandonedStream (:1140-1143): marked now, dropped by the ClearAbandonedStreams of the connection's next client parse
__global__ void k_h2_client_abandon(H2Conn* conns, uint32_t conn, const uint32_t* ids, uint32_t n, H2Pool pool) {
    if (!(conns[conn].pad0 & kH2ClientMode)) return;
    H2Stream* S = pool.streams + (size_t)conn * pool.pending;
    for (uint32_t i = 0; i < n; i++) { const int k = h2_find(S, pool.pending, (int32_t)ids[i]); if (k >= 0) S[k].stream_ended |= kH2Abandoned; }
}
__device__ __forceinline__ int32_t h2c_status_of_error(uint32_t e) {                     // H2ErrorToStatusCode (http2.cpp:88-112)
    switch (e) {
    case 0: return 200;
    case 4: return 504;
    case 5: return 400;
    case 7: case 8: case 11: return 503;
    case 12: return 401;
    case 13: return 505;
    default: return 500;
    }
}
// strtol(c_str, NULL, 10) cast to int: leading white space, a sign, digits; saturates at LONG_MIN / LONG_MAX like glibc
__device__ __forceinline__ int32_t h2c_strtol(const uint8_t* v, uint32_t vl) {
    const uint32_t m = cstr_len(v, vl);
    uint32_t i = 0;
    while (i < m && (v[i] == ' ' || (v[i] >= 9 && v[i] <= 13))) i++;
    bool neg = false;
    if (i < m && (v[i] == '+' || v[i] == '-')) { neg = v[i] == '-'; i++; }
    unsigned long long acc = 0; bool sat = false;
    for (; i < m && v[i] >= '0' && v[i] <= '9'; i++) {
        if (acc > (0x7fffffffffffffffull - (v[i] - '0')) / 10) sat = true;
        else acc = acc * 10 + (v[i] - '0');
    }
    long long r = sat ? (neg ? (long long)0x8000000000000000ull : 0x7fffffffffffffffll) : (neg ? -(long long)acc : (long long)acc);
    return (int32_t)(uint32_t)(unsigned long long)r;
}
__device__ __forceinline__ int32_t h2c_grpc_errno(int32_t s) {                           // GrpcStatusToErrorCode (grpc.cpp:83-125)
    switch (s) {
    case 0: return 0;
    case 1: return 125;                                          // ECANCELED
    case 3: return 22;                                           // EINVAL
    case 4: return 1008;                                         // ERPCTIMEDOUT
    case 6: return 17;                                           // EEXIST
    case 7: return 1;                                            // EPERM
    case 8: return 2004;                                         // ELIMIT
    case 12: return 1002;                                        // ENOMETHOD
    case 16: return 1004;                                        // ERPCAUTH
    default: return 2001;                                        // EINTERNAL
    }
}
__device__ __forceinline__ const char* h2c_grpc_name(int32_t s) {                         // GrpcStatusToString (grpc.cpp:29-51)
    const char* const names[18] = { "GRPC_OK", "GRPC_CANCELED", "GRPC_UNKNOWN", "GRPC_INVALIDARGUMENT", "GRPC_DEADLINEEXCEEDED", "GRPC_NOTFOUND",
        "GRPC_ALREADYEXISTS", "GRPC_PERMISSIONDENIED", "GRPC_RESOURCEEXHAUSTED", "GRPC_FAILEDPRECONDITION", "GRPC_ABORTED", "GRPC_OUTOFRANGE",
        "GRPC_UNIMPLEMENTED", "GRPC_INTERNAL", "GRPC_UNAVAILABLE", "GRPC_DATALOSS", "GRPC_UNAUTHENTICATED", "GRPC_MAX" };
    return (s >= 0 && s < 18) ? names[s] : "Unknown-GrpcStatus";
}
__device__ __forceinline__ const char* h2c_reason(int32_t sc) {                           // HttpReasonPhrase (http_status_code.cpp:27-115)
    switch (sc) {
    case 100: return "Continue"; case 101: return "Switching Protocols";
    case 200: return "OK"; case 201: return "Created"; case 202: return "Accepted"; case 203: return "Non-Authoritative Informational";
    case 204: return "No Content"; case 205: return "Reset Content"; case 206: return "Partial Content";
    case 300: return "Multiple Choices"; case 301: return "Move Permanently"; case 302: return "Found"; case 303: return "See Other";
    case 304: return "Not Modified"; case 305: return "Use Proxy"; case 307: return "Temporary Redirect";
    case 400: return "Bad Request"; case 401: return "Unauthorized"; case 402: return "Payment Required"; case 403: return "Forbidden";
    case 404: return "Not Found"; case 405: return "Method Not Allowed"; case 406: return "Not Acceptable";
    case 407: return "Proxy Authentication Required"; case 408: return "Request Timeout"; case 409: return "Conflict"; case 410: return "Gone";
    case 411: return "Length Required"; case 412: return "Precondition Failed"; case 413: return "Request Entity Too Large";
    case 414: return "Request-URI Too Long"; case 415: return "Unsupported Media Type"; case 416: return "Requested Range Not Satisfiable";
    case 417: return "Expectation Failed";
    case 500: return "Internal Server Error"; case 501: return "Not Implemented"; case 502: return "Bad Gateway"; case 503: return "Service Unavailable";
    case 504: return "Gateway Timeout"; case 505: return "HTTP Version Not Supported";
    default: return nullptr;                                     // "Unknown status code (%d)"
    }
}
__device__ __forceinline__ uint32_t h2c_hex(uint8_t c) {                                   // hex_to_int (grpc.cpp:143-152)
    return (c >= 'a' && c <= 'f') ? c - 'a' + 10u : (c >= 'A' && c <= 'F') ? c - 'A' + 10u : (c >= '0' && c <= '9') ? c - '0' : 0u;
}
// PercentDecode (grpc.cpp:154-170) of v[0..vl) into dst (NULL: length only); SetFailed("%s", decoded.c_str()) stops at the first NUL
__device__ __forceinline__ uint32_t h2c_percent_decode(const uint8_t* v, uint32_t vl, uint8_t* dst) {
    uint32_t o = 0;
    for (uint32_t i = 0; i < vl; i++) {
        uint8_t ch = v[i];
        if (ch == '%' && i + 2 < vl) { ch = (uint8_t)(h2c_hex(v[i + 1]) * 16 + h2c_hex(v[i + 2])); i += 2; }
        if (ch == 0) break;
        if (dst) dst[o] = ch;
        o++;
    }
    return o;
}
// the record of header `name` in the MERGED list (what HttpHeader::GetHeader sees): value pointer and length, false if absent.  GetHeader
// compares case-insensitively; an exact compare is the same here because HPacker::Decode lowercases every name (hpack.cpp:755) and the
// decoder above does too, so no upper-case name reaches the records
__device__ __forceinline__ bool h2c_get(const uint8_t* recs, uint32_t len, const char* name, const uint8_t*& v, uint32_t& vl) {
    for (uint32_t q = 0; q < len;) {
        const uint32_t nl = recs[q] | ((uint32_t)recs[q + 1] << 8), l2 = recs[q + 2] | ((uint32_t)recs[q + 3] << 8);
        if (lit_eq(recs + q + 4, cstr_len(recs + q + 4, nl), name)) { v = recs + q + 4 + nl; vl = l2; return true; }
        q += 4 + nl + l2;
    }
    return false;
}
__device__ __forceinline__ bool h2c_name_eq(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {   // case-insensitive, as c_str
    an = cstr_len(a, an); bn = cstr_len(b, bn);
    if (an != bn) return false;
    for (uint32_t i = 0; i < an; i++) if (lc(a[i]) != lc(b[i])) return false;
    return true;
}
// The stream's decoded fields (every record, pseudo-headers included, in wire order) folded the way ConsumeHeaders fills HttpHeader
// (:1233-1288): ":status" -> status_code (strtol, last one wins), "content-type" -> set_content_type (the last value wins, one record at
// the place of the first), "set-cookie" -> one record each (AddHeader), every other name -> AppendHeader (http_header.cpp:100-117): the
// first record of a name (case-insensitive) takes the values of all later ones, joined with "," ("; " for "cookie"), an empty value is
// replaced instead of joined.  brpc's header map has no order; the records here keep the order in which names first appear.
__device__ __forceinline__ uint32_t h2c_merge(const uint8_t* raw, uint32_t raw_len, uint8_t* out, uint32_t& n_out, int32_t& status) {
    uint32_t o = 0; n_out = 0;
    for (uint32_t q = 0; q < raw_len;) {
        const uint32_t nl = raw[q] | ((uint32_t)raw[q + 1] << 8), vl = raw[q + 2] | ((uint32_t)raw[q + 3] << 8);
        const uint8_t* nm = raw + q + 4; const uint8_t* v = nm + nl;
        const uint32_t cn = cstr_len(nm, nl);
        const uint32_t next = q + 4 + nl + vl;
        if (cn && nm[0] == ':') {
            if (lit_eq(nm, cn, ":status")) status = h2c_strtol(v, vl);
            q = next; continue;
        }
        const bool ct = lit_eq(nm, cn, "content-type"), cookie_set = h2c_name_eq(nm, nl, (const uint8_t*)"set-cookie", 10);
        bool first = true;
        if (!cookie_set) for (uint32_t p = 0; p < q && first;) {   // an earlier record of the same header already took this one
            const uint32_t pl = raw[p] | ((uint32_t)raw[p + 1] << 8), pv = raw[p + 2] | ((uint32_t)raw[p + 3] << 8);
            const uint8_t* pn = raw + p + 4;
            const uint32_t pc = cstr_len(pn, pl);
            if (!(pc && pn[0] == ':')) {
                if (ct) { if (lit_eq(pn, pc, "content-type")) first = false; }
                else if (!lit_eq(pn, pc, "content-type") && h2c_name_eq(pn, pl, nm, nl)) first = false;
            }
            p += 4 + pl + pv;
        }
        if (!first) { q = next; continue; }
        uint8_t* rec = out + o;
        for (uint32_t i = 0; i < nl; i++) rec[4 + i] = nm[i];
        uint32_t ol = 0;
        uint8_t* val = rec + 4 + nl;
        if (cookie_set) { for (uint32_t i = 0; i < vl; i++) val[i] = v[i]; ol = vl; }
        else {
            const bool semi = h2c_name_eq(nm, nl, (const uint8_t*)"cookie", 6);
            for (uint32_t p = q; p < raw_len;) {
                const uint32_t pl = raw[p] | ((uint32_t)raw[p + 1] << 8), pv = raw[p + 2] | ((uint32_t)raw[p + 3] << 8);
                const uint8_t* pn = raw + p + 4; const uint8_t* pvp = pn + pl;
                const uint32_t pc = cstr_len(pn, pl);
                const bool same = !(pc && pn[0] == ':') && (ct ? lit_eq(pn, pc, "content-type") : (!lit_eq(pn, pc, "content-type") && h2c_name_eq(pn, pl, nm, nl)));
                if (same) {
                    if (ct || ol == 0) { for (uint32_t i = 0; i < pv; i++) val[i] = pvp[i]; ol = pv; }
                    else {
                        if (semi) { val[ol++] = ';'; val[ol++] = ' '; } else val[ol++] = ',';
                        for (uint32_t i = 0; i < pv; i++) val[ol + i] = pvp[i];
                        ol += pv;
                    }
                }
                p += 4 + pl + pv;
            }
        }
        rec[0] = (uint8_t)nl; rec[1] = (uint8_t)(nl >> 8); rec[2] = (uint8_t)ol; rec[3] = (uint8_t)(ol >> 8);
        o += 4 + nl + ol; n_out++;
        q = next;
    }
    return o;
}
__device__ __forceinline__ uint32_t h2c_puts(uint8_t* dst, uint32_t o, const char* s) { for (uint32_t i = 0; s[i]; i++) { if (dst) dst[o] = (uint8_t)s[i]; o++; } return o; }
__device__ __forceinline__ uint32_t h2c_putd(uint8_t* dst, uint32_t o, int32_t v) {
    uint8_t tmp[12]; const uint32_t n = put_dec_i32_h2(tmp, v);
    for (uint32_t i = 0; i < n; i++) { if (dst) dst[o] = tmp[i]; o++; }
    return o;
}
// ProcessHttpResponse's decisions for a protobuf-typed call (http_rpc_protocol.cpp:390-533, up to the body parse): the error code and the
// text SetFailed receives (written to dst unless NULL), from the merged header records and the body (gRPC: without its prefix)
__device__ __forceinline__ uint32_t h2c_verdict(const uint8_t* recs, uint32_t rlen, int32_t sc, bool is_grpc, bool prefix_ok, bool compressed,
                                                const uint8_t* body, uint32_t body_len, int32_t grpc_status, bool has_grpc_status,
                                                uint8_t* dst, int32_t& code) {
    code = 0;
    if (is_grpc) {
        if (!prefix_ok) { code = 2002; return h2c_puts(dst, 0, "Invalid gRPC response"); }                      // ERESPONSE
        if (has_grpc_status && grpc_status != 0) {
            code = h2c_grpc_errno(grpc_status);
            const uint8_t* m; uint32_t ml;
            if (h2c_get(recs, rlen, "grpc-message", m, ml)) return h2c_percent_decode(m, ml, dst);
            return h2c_puts(dst, 0, h2c_grpc_name(grpc_status));
        }
    }
    if (sc < 200 || sc >= 300) {                                 // EHTTP, "HTTP/%d.%d %d %s[: body]" then "%s" of its c_str
        code = 1010;
        uint32_t o = h2c_puts(dst, 0, "HTTP/2.0 ");
        o = h2c_putd(dst, o, sc);
        if (dst) dst[o] = ' ';
        o++;
        const char* rp = h2c_reason(sc);
        if (rp) o = h2c_puts(dst, o, rp);
        else { o = h2c_puts(dst, o, "Unknown status code ("); o = h2c_putd(dst, o, sc); o = h2c_puts(dst, o, ")"); }
        if (body_len) {
            o = h2c_puts(dst, o, ": ");
            const uint32_t k = body_len < kH2ErrMax ? body_len : kH2ErrMax;
            for (uint32_t i = 0; i < k && body[i]; i++) { if (dst) dst[o] = body[i]; o++; }
        }
        return o;
    }
    if (is_grpc && compressed) {
        const uint8_t* e; uint32_t el;
        if (!h2c_get(recs, rlen, "grpc-encoding", e, el)) { code = 2002; return h2c_puts(dst, 0, "Fail to find header `grpc-encoding' in compressed gRPC response"); }
    }
    return 0;
}

// ClearAbandonedStreams (:1145-1157): ParseH2Message runs it each time it returns, i.e. after every frame that produced a message and
// when the input ends; RemoveStreamAndDeferWU of each, here in ascending id order (brpc pops the most recent first)
__device__ __forceinline__ void h2c_clear_abandoned(H2Conn& c, H2Stream* S, uint32_t P, H2Out& o) {
    for (;;) {
        int best = -1;
        for (uint32_t i = 0; i < P; i++) if (S[i].id >= 0 && (S[i].stream_ended & kH2Abandoned) && (best < 0 || S[i].id < S[best].id)) best = (int)i;
        if (best < 0) break;
        (void)h2_remove_stream(c, S, P, o, S[best].id);
    }
}
// a header block of a stream the client does not know, decoded into a throw-away stream at the end of the blob so that the HPACK table
// advances, then dropped
__device__ __forceinline__ int h2c_discard_headers(H2Conn& c, HpackState& hp, H2Out& o, const uint8_t* frag, uint32_t n, bool& no_room) {
    if (o.blob_off + kH2HdrBytes > o.blob_end) { no_room = true; return -1; }
    H2Stream tmp; tmp.hdr_len = 0; tmp.n_headers = 0;
    return h2_consume_headers(c, hp, tmp, o.base + o.blob_end - kH2HdrBytes, frag, n, no_room);
}
// The stream (already out of the pending map; its bytes are still in `slot`) leaves a client connection as one b2_h2_call, with what
// ProcessHttpResponse decides before the body is parsed.  False when the run's descriptors or blob space ran out.
__device__ __forceinline__ bool h2_emit_call(const H2Stream& st, const uint8_t* slot, int32_t sid, uint32_t how, int32_t status_override, uint32_t r,
                                             uint32_t gbase, H2Out& o, const uint8_t* bytes, b2_h2_call* cout, uint32_t& n_calls, uint32_t cap) {
    const bool in_input = st.body_input_off != 0;
    const uint32_t need1 = ((st.hdr_len + 15u) & ~15u) + (in_input ? 0u : ((st.body_len + 15u) & ~15u));
    if (n_calls >= cap || o.blob_off + need1 > o.blob_end) return false;
    const uint32_t ho = o.blob_off, bo = ho + ((st.hdr_len + 15u) & ~15u), eo = o.blob_off + need1;
    b2_h2_call m;
    m.run_idx = r; m.stream_id = (uint32_t)sid; m.how = how; m.flags = 0;
    int32_t sc = 200;                                            // HttpHeader() (http_header.cpp:30)
    uint32_t nh = 0;
    const uint32_t ml = h2c_merge(slot, st.hdr_len, o.base + ho, nh, sc);
    if (status_override >= 0) sc = status_override;
    if (!in_input) thread_copy(o.base + bo, slot + kH2HdrBytes, st.body_len);
    m.headers_off = gbase + ho; m.headers_len = ml; m.n_headers = nh;
    m.body_off = in_input ? st.body_input_off : gbase + bo; m.body_len = st.body_len;
    if (in_input) m.flags |= B2_H2_FLAG_BODY_IN_INPUT;
    const uint8_t* body_p = in_input ? bytes + st.body_input_off : o.base + bo;
    m.status_code = sc;
    const uint8_t* recs = o.base + ho;
    const uint8_t* v; uint32_t vl;
    bool is_grpc = false;
    if (h2c_get(recs, ml, "content-type", v, vl)) (void)h2_content_type(v, cstr_len(v, vl), is_grpc);
    bool prefix_ok = false, compressed = false;
    const uint8_t* msg_p = body_p; uint32_t msg_len = st.body_len;
    m.msg_off = 0; m.msg_len = 0;
    if (is_grpc) {
        m.flags |= B2_H2_FLAG_GRPC;
        const H2GrpcMsg g = h2_remove_grpc_prefix(body_p, st.body_len, m.body_off);
        prefix_ok = g.prefix_ok; compressed = g.compressed; m.msg_off = g.msg_off; m.msg_len = g.msg_len;
        if (prefix_ok) { m.flags |= B2_H2_FLAG_GRPC_PREFIX_OK; msg_p = body_p + (st.body_len ? 5 : 0); msg_len = m.msg_len; }
        if (compressed) m.flags |= B2_H2_FLAG_GRPC_COMPRESSED;
    }
    const bool has_gs = h2c_get(recs, ml, "grpc-status", v, vl);
    m.grpc_status = has_gs ? h2c_strtol(v, vl) : -1;
    if (has_gs) m.flags |= B2_H2_CALL_HAS_GRPC_STATUS;
    int32_t code = 0;
    const uint32_t el = h2c_verdict(recs, ml, sc, is_grpc, prefix_ok, compressed, msg_p, msg_len, m.grpc_status, has_gs, nullptr, code);
    if (eo + ((el + 15u) & ~15u) > o.blob_end) return false;
    (void)h2c_verdict(recs, ml, sc, is_grpc, prefix_ok, compressed, msg_p, msg_len, m.grpc_status, has_gs, o.base + eo, code);
    m.error_code = code; m.error_off = el ? gbase + eo : 0; m.error_len = el;
    o.blob_off = eo + ((el + 15u) & ~15u);
    cout[n_calls++] = m;
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// H2Context::Consume (:467-543) over one connection run, for the server (k_h2_consume: every request becomes a b2_h2_msg) or the client
// (k_h2_client_consume: every stream that leaves the connection becomes a b2_h2_call).  Like the reference it is one body; the side is
// a template argument and each `if constexpr (kClient)` sits where brpc asks is_server_side() / is_client_side().
template <bool kClient>
__device__ __forceinline__ void h2_consume_run(uint32_t r, const uint8_t* bytes, const b2_run* runs, H2Conn* conns, HpackState* hps,
                                               const DevMethod* methods, uint32_t n_methods, b2_h2_run_status* rs,
                                               typename std::conditional<kClient, b2_h2_call, b2_h2_msg>::type* descs, uint32_t cap_per_run,
                                               uint8_t* out, uint32_t region, H2Pool pool) {
    const uint32_t conn = (uint32_t)runs[r].socket_id;
    const uint32_t P = pool.pending, kH2StreamBytes = pool.stream_bytes;
    H2Stream* const S = pool.streams + (size_t)conn * P;
    uint8_t* const slots = pool.slots + (size_t)conn * P * kH2StreamBytes;
    const uint32_t run_off = runs[r].offset;
    const uint8_t* in = bytes + run_off; const uint32_t n = runs[r].length;
    H2Conn& c = conns[conn];
    HpackState& hp = hps[conn];
    H2Out o; o.base = out + (size_t)r * region; o.ctrl_cap = region / 4; o.ctrl_len = 0; o.blob_off = region / 4; o.blob_end = region; o.overflow = false;
    auto* const dout = descs + (size_t)r * cap_per_run;
    const uint32_t gbase = r * region;
    uint32_t n_out = 0, pos = 0, last_ok = 0, perr = B2_PARSE_ERROR_NOT_ENOUGH_DATA;
    bool no_room = false;
    if constexpr (kClient) {
        if (!(c.pad0 & kH2ClientMode)) {                         // not a client connection: nothing is read, nothing changes
            b2_h2_run_status st; st.consumed = 0; st.parse_error = B2_PARSE_ERROR_TRY_OTHERS; st.n_msgs = 0; st.first_msg = 0;
            st.ctrl_off = r * region; st.ctrl_len = 0; st.remote_max_frame_size = 0; st.remote_stream_window_size = 0;
            rs[r] = st;
            return;
        }
    }
    // the stream in slot k (out of the pending map already) leaves the connection as this side's descriptor; `how` and `status` are
    // the client's (how the call ended, a status that replaces the stream's :status, or -1)
    auto emit = [&](int k, int32_t sid, uint32_t how, int32_t status) -> bool {
        if constexpr (kClient) return h2_emit_call(S[k], slots + (size_t)k * kH2StreamBytes, sid, how, status, r, gbase, o, bytes, dout, n_out, cap_per_run);
        else return h2_emit_msg(S[k], slots + (size_t)k * kH2StreamBytes, sid, r, gbase, o, bytes, methods, n_methods, dout, n_out, cap_per_run);
    };
    uint32_t n_cleared = 0;                                      // client: n_out when abandoned streams were last cleared
    for (;;) {
        if constexpr (kClient) {
            if (n_out != n_cleared) { h2c_clear_abandoned(c, S, P, o); n_cleared = n_out; }   // the previous frame returned a message
        }
        if (o.overflow || no_room) { perr = B2_PARSE_ERROR_NO_RESOURCE; break; }
        if (c.conn_state == 0) {                                 // H2_CONNECTION_UNINITIALIZED (:469-492)
            if constexpr (kClient) { c.conn_state = 1; last_ok = pos; continue; }   // client side: READY without reading a preface
            else {
                const char* pre = "PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n";
                const uint32_t k = (n - pos) < 24 ? (n - pos) : 24;
                bool match = true;
                for (uint32_t i = 0; i < k; i++) if (in[pos + i] != (uint8_t)pre[i]) { match = false; break; }
                if (!match) { perr = B2_PARSE_ERROR_TRY_OTHERS; break; }
                if (k < 24) break;
                c.conn_state = 1; pos += 24;
                // SerializeH2SettingsFrameAndWU of the default server settings (:230-259): ENABLE_PUSH=0, INITIAL_WINDOW_SIZE=256K, WU 1M-65535
                uint8_t* p = h2_ack_room(o, 9 + 12 + 13);
                if (p) {
                    h2_put_head(p, 12, 4, 0, 0);
                    p[9] = 0; p[10] = 2; put_be32(p + 11, 0);
                    p[15] = 0; p[16] = 4; put_be32(p + 17, c.l_stream_window_size);
                    h2_put_head(p + 21, 4, 8, 0, 0); put_be32(p + 30, 1024 * 1024 - 65535);
                }
                last_ok = pos;
                continue;
            }
        }
        // ---- ConsumeFrameHead (:438-465)
        const uint32_t left = n - pos;
        if (left < 3) break;
        const uint32_t length = ((uint32_t)in[pos] << 16) | ((uint32_t)in[pos + 1] << 8) | in[pos + 2];
        if (length > c.l_max_frame_size) { perr = B2_PARSE_ERROR_ABSOLUTELY_WRONG; break; }
        if ((unsigned long long)(left - 3) < 6ull + length) break;
        const uint32_t type = in[pos + 3], flags = in[pos + 4], sid_raw = load_be32(in + pos + 5);
        if (sid_raw & 0x80000000u) { perr = B2_PARSE_ERROR_ABSOLUTELY_WRONG; break; }
        const int32_t sid = (int32_t)sid_raw;
        pos += 9;
        if (type > 9) { perr = B2_PARSE_ERROR_ABSOLUTELY_WRONG; break; }          // FindFrameHandler == NULL (:498-502)
        const uint8_t* pl = in + pos;                                // payload; handlers advance `used`
        uint32_t used = 0;
        H2Res res = h2_ok();
        uint32_t how = B2_H2_CALL_ENDED; int32_t sc_over = -1;       // client: how a stream that leaves ends, and its status
        bool goaway = false; int32_t goaway_last = 0;                // client: a GOAWAY was read, and its last_stream_id
        switch (type) {
        case 0: {                                                    // ---- OnData (:699-726) + H2StreamContext::OnData (:728-779)
            uint32_t frag = length, padl = 0;
            if ((flags & 0x8) && length == 0) { res = h2_err(6); break; }   // no room for the pad-length byte (the reference would read past the frame)
            if (flags & 0x8) { frag--; padl = pl[used++]; }
            if (frag < padl) { res = h2_err(6); break; }
            frag -= padl;
            const int k = h2_find(S, P, sid);
            if (k < 0) {
                // stream unknown: the bytes are still counted against the connection window, then STREAM_CLOSED
                used += frag + padl;
                long long tmp_deferred = 0;
                (void)h2_data_quota(c, o, sid, tmp_deferred, frag);  // (the FLOW_CONTROL result of the throw-away stream is discarded)
                h2_defer_wu(c, o, tmp_deferred);
                res = h2_err(5, sid);
                break;
            }
            H2Stream& st = S[k];
            if (st.body_len == 0 && (flags & 0x1) && frag) {
                // the usual unary call: one DATA frame that also ends the stream — the body stays where it is in the batch
                st.body_input_off = run_off + pos + used; st.body_len = frag;
            } else {
                if (kH2HdrBytes + st.body_len + frag > kH2StreamBytes) { no_room = true; break; }
                thread_copy(slots + (size_t)k * kH2StreamBytes + kH2HdrBytes + st.body_len, pl + used, frag);
                st.body_len += frag;
            }
            used += frag + padl;
            if (!h2_data_quota(c, o, sid, st.deferred_wu, frag)) { res = h2_err(3, sid); break; }
            if (flags & 0x1) res = h2_end_stream(c, S, P, o, sid);
            break; }
        case 1: {                                                    // ---- OnHeaders (:545-614) + H2StreamContext::OnHeaders (:616-653)
            if (sid == 0) { res = h2_err(1); break; }
            const bool has_padding = flags & 0x8, has_priority = flags & 0x20;
            if (length < (has_priority ? 5u : 0u) + (has_padding ? 1u : 0u)) { res = h2_err(6); break; }
            uint32_t frag = length, padl = 0;
            if (has_padding) { padl = pl[used++]; frag--; }
            if (has_priority) { used += 5; frag -= 5; }
            if (frag < padl) { res = h2_err(6); break; }
            frag -= padl;
            int k;
            if constexpr (kClient) {
                k = h2_find(S, P, sid);
                if (k < 0) {
                    // unknown stream (:600-606); a failed decode leaves the rest of the payload unread, as the throw-away OnHeaders
                    // returns before moving the iterator
                    if (h2c_discard_headers(c, hp, o, pl + used, frag, no_room) == 0) used += frag + padl;
                    break;
                }
            } else if (sid > c.last_received_stream_id) {            // new stream (:578-596)
                if ((sid & 1) == 0) { res = h2_err(1); break; }
                c.last_received_stream_id = sid;
                k = h2_find(S, P, -1);
                if (k < 0) { no_room = true; break; }                // (device limit: B2_H2_MAX_PENDING)
                H2Stream& st = S[k];
                st.id = sid; st.hdr_len = 0; st.n_headers = 0; st.body_len = 0; st.stream_ended = 0; st.deferred_wu = 0; st.body_input_off = 0;
                st.remote_window_left = (long long)c.r_stream_window_size;
                c.n_pending++;
            } else {
                k = h2_find(S, P, sid);
                if (k < 0) { res = h2_err(1); break; }
            }
            H2Stream& st = S[k];
            if (h2_consume_headers(c, hp, st, slots + (size_t)k * kH2StreamBytes, pl + used, frag, no_room) < 0) { if (!no_room) res = h2_err(1); break; }
            used += frag + padl;
            if (flags & 0x4) { if (flags & 0x1) res = h2_end_stream(c, S, P, o, sid); }
            else if (flags & 0x1) {                                  // END_STREAM before END_HEADERS: CONTINUATION ends the stream
                if constexpr (kClient) st.stream_ended |= 1u;        // (client streams also carry kH2Abandoned there)
                else st.stream_ended = 1;
            }
            break; }
        case 2: res = h2_err(1); break;                              // OnPriority (:918-922)
        case 3: {                                                    // ---- OnResetStream (:781-823)
            if (length != 4) { res = h2_err(6); break; }
            used += 4;
            if constexpr (kClient) {                                 // client side: the stream leaves as a call (:815-820)
                const uint32_t e = load_be32(pl);
                const int k = h2_remove_stream(c, S, P, o, sid);
                if (k >= 0) { res.kind = 1; res.slot = k; res.err_stream = sid; how = B2_H2_CALL_RESET_BY_PEER; sc_over = h2c_status_of_error(e); }
            } else (void)h2_remove_stream(c, S, P, o, sid);        // server side: the stream is dropped, no message
            break; }
        case 4: {                                                    // ---- OnSettings (:848-916)
            if (sid != 0) { res = h2_err(1); break; }
            if (flags & 0x1) {
                if (length != 0) { res = h2_err(1); break; }
                if constexpr (kClient) { c.l_stream_window_size = 256 * 1024; c.l_max_frame_size = 16384; }   // _local_settings = _unack_local_settings
                break;
            }
            const long long old_sw = (long long)c.r_stream_window_size;
            uint32_t t_hts, t_push, t_mcs, t_sws, t_mfs, t_mhl;
            if (!c.remote_settings_received) { t_hts = 4096; t_push = 0; t_mcs = 0xffffffffu; t_sws = 256 * 1024; t_mfs = 16384; t_mhl = 0xffffffffu; }
            else { t_hts = c.r_header_table_size; t_push = c.r_enable_push; t_mcs = c.r_max_concurrent_streams; t_sws = c.r_stream_window_size; t_mfs = c.r_max_frame_size; t_mhl = c.r_max_header_list_size; }
            bool okp = (length / 6) * 6 == length;                   // ParseH2Settings (:166-211)
            if (okp) for (uint32_t i = 0; i < length / 6; i++) {
                const uint32_t id = ((uint32_t)pl[used] << 8) | pl[used + 1], value = load_be32(pl + used + 2);
                used += 6;
                if (id == 1) t_hts = value;
                else if (id == 2) { if (value > 1) { okp = false; break; } t_push = value; }
                else if (id == 3) t_mcs = value;
                else if (id == 4) { if (value > (uint32_t)kH2MaxWindow) { okp = false; break; } t_sws = value; }
                else if (id == 5) { if (value > 16777215u || value < 16384u) { okp = false; break; } t_mfs = value; }
                else if (id == 6) t_mhl = value;
            }
            if (!c.remote_settings_received) {
                if (!okp) { res = h2_err(1); break; }                // parsed into a temporary: nothing is kept
                c.remote_window_left -= (kH2MaxWindow - 65535);
                c.remote_settings_received = 1;
            }
            // (after the first frame the reference parses in place: fields set before a bad pair stay)
            c.r_header_table_size = t_hts; c.r_enable_push = t_push; c.r_max_concurrent_streams = t_mcs;
            c.r_stream_window_size = t_sws; c.r_max_frame_size = t_mfs; c.r_max_header_list_size = t_mhl;
            if (!okp) { res = h2_err(1); break; }
            const long long diff = (long long)c.r_stream_window_size - old_sw;
            bool flow_ok = true;
            if (diff) for (uint32_t i = 0; i < P; i++) if (S[i].id >= 0) { if (!h2_add_window(S[i].remote_window_left, diff)) { flow_ok = false; break; } }
            if (!flow_ok) { res = h2_err(3); break; }
            uint8_t* p = h2_ack_room(o, 9); if (p) h2_put_head(p, 0, 4, 1, 0);
            break; }
        case 5: res = h2_err(1); break;                              // OnPushPromise (:924-928)
        case 6: {                                                    // ---- OnPing (:930-952)
            if (length != 8) { res = h2_err(6); break; }
            if (sid != 0) { res = h2_err(1); break; }
            if (flags & 0x1) break;                                  // (an ack's payload is left unread, as in the reference)
            uint8_t* p = h2_ack_room(o, 17);
            if (p) { h2_put_head(p, 8, 6, 1, 0); for (uint32_t i = 0; i < 8; i++) p[9 + i] = pl[i]; }
            used += 8;
            break; }
        case 7: {                                                    // ---- OnGoAway (:959-1006): the server ignores it
            if (length < 8) { res = h2_err(6); break; }
            if (sid != 0) { res = h2_err(1); break; }
            if (flags) { res = h2_err(1); break; }
            if constexpr (kClient) { goaway_last = (int32_t)load_be32(pl + length - 8); goaway = true; }   // (:979-1003) after the debug data
            used += length;
            break; }
        case 8: {                                                    // ---- OnWindowUpdate (:1008-1038)
            if (length != 4) { res = h2_err(6); break; }
            const uint32_t inc = load_be32(pl); used += 4;
            if ((inc & 0x80000000u) || inc == 0) { res = h2_err(1); break; }
            if (sid == 0) { if (!h2_add_window(c.remote_window_left, (long long)inc)) res = h2_err(3); break; }
            const int k = h2_find(S, P, sid);
            if (k < 0) break;
            if (!h2_add_window(S[k].remote_window_left, (long long)inc)) res = h2_err(3);
            break; }
        case 9: {                                                    // ---- OnContinuation (:655-697)
            const int k = h2_find(S, P, sid);
            if (k < 0) {
                if constexpr (kClient) {                             // unknown stream: decoded and dropped (:659-665)
                    used += length;
                    (void)h2c_discard_headers(c, hp, o, pl, length, no_room);
                } else res = h2_err(1);
                break;
            }
            H2Stream& st = S[k];
            used += length;                                          // the payload moves into _remaining_header_fragment first
            if (h2_consume_headers(c, hp, st, slots + (size_t)k * kH2StreamBytes, pl, length, no_room) < 0) { if (!no_room) res = h2_err(1); break; }
            if ((flags & 0x4) && (kClient ? (st.stream_ended & 1u) : st.stream_ended)) res = h2_end_stream(c, S, P, o, sid);
            break; }
        }
        if (no_room) continue;
        pos += used;
        if (res.kind == 2) {
            if (res.err_stream) {                                    // RST_STREAM, then the stream is forgotten (:508-528)
                uint8_t* p = h2_ack_room(o, 13);
                if (p) { h2_put_head(p, 4, 3, 0, (uint32_t)res.err_stream); put_be32(p + 9, res.err); }
                if constexpr (kClient) {                             // a stream of ours leaves as a call (:519-526)
                    const int k = h2_remove_stream(c, S, P, o, res.err_stream);
                    if (k >= 0 && !emit(k, res.err_stream, B2_H2_CALL_RESET_BY_US, h2c_status_of_error(res.err))) no_room = true;
                } else (void)h2_remove_stream(c, S, P, o, res.err_stream);
            } else {                                                 // GOAWAY (:529-538); parsing goes on
                // (the client's _last_received_stream_id stays -1: H2Conn::last_received_stream_id holds its _goaway_stream_id)
                uint8_t* p = h2_ack_room(o, 17);
                if (p) { h2_put_head(p, 8, 7, 0, 0); put_be32(p + 9, kClient ? 0xffffffffu : (uint32_t)c.last_received_stream_id); put_be32(p + 13, res.err); }
            }
            last_ok = pos;
            continue;
        }
        last_ok = pos;
        if constexpr (kClient) {
            if (goaway) {
                // SetLogOff + RemoveGoAwayStreams (:388-414): _goaway_stream_id = last; the streams above it (all of them for 0) leave with
                // status 503, without moving their deferred WINDOW_UPDATE (erase, not RemoveStreamAndDeferWU).  brpc walks its map in
                // hash order; the calls here come in ascending stream id order.
                c.last_received_stream_id = goaway_last;
                for (;;) {
                    int best = -1;
                    for (uint32_t i = 0; i < P; i++)                 // (free records have id -1: a last_stream_id >= 2^31 is negative here)
                        if (S[i].id >= 0 && S[i].id > goaway_last && (best < 0 || S[i].id < S[best].id)) best = (int)i;
                    if (best < 0) break;
                    const int32_t gid = S[best].id;
                    S[best].id = -1; c.n_pending--;
                    if (!emit(best, gid, B2_H2_CALL_GOAWAY, 503)) { no_room = true; break; }
                }
                continue;
            }
        }
        if (res.kind == 1 && !emit(res.slot, res.err_stream, how, sc_over)) no_room = true;
    }
    if constexpr (kClient) {
        h2c_clear_abandoned(c, S, P, o);
        if (o.overflow) perr = B2_PARSE_ERROR_NO_RESOURCE;
    }
    b2_h2_run_status st; st.consumed = last_ok; st.parse_error = perr; st.n_msgs = n_out; st.first_msg = o.blob_off - region / 4;      // blob bytes used (the host turns this field into the list index)
    st.ctrl_off = r * region; st.ctrl_len = o.ctrl_len; st.remote_max_frame_size = c.r_max_frame_size; st.remote_stream_window_size = c.r_stream_window_size;
    rs[r] = st;
}
__global__ void k_h2_consume(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, H2Conn* conns, HpackState* hps,
                             const DevMethod* methods, uint32_t n_methods, b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t msg_cap_per_run,
                             uint8_t* out, uint32_t region, H2Pool pool) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_runs) return;
    h2_consume_run<false>(r, bytes, runs, conns, hps, methods, n_methods, rs, msgs, msg_cap_per_run, out, region, pool);
}
__global__ void k_h2_client_consume(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, H2Conn* conns, HpackState* hps,
                                    b2_h2_run_status* rs, b2_h2_call* calls, uint32_t call_cap_per_run, uint8_t* out, uint32_t region, H2Pool pool) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_runs) return;
    h2_consume_run<true>(r, bytes, runs, conns, hps, nullptr, 0, rs, calls, call_cap_per_run, out, region, pool);
}

// ---------------------------------------------------------------------------------------------------------
// gzip-compressed messages on connections opted in with b2_h2_conn_set_gunzip: the step of ProcessHttpRequest (policy/http_rpc_protocol.cpp
// :1645-1683) / ProcessHttpResponse (:507-529) between RemoveGrpcPrefix and the protobuf parse, over what h2_consume_run left
// on the device.  Four passes, launched only when a run of the batch is on such a connection:
//   select (one thread per run: the server's raw records are merged like the client's) -> size (one thread per candidate,
//   gz_input_stream<false>) -> place (one thread per run, message order, 16-byte aligned after the parse's own bytes in the run's region)
//   -> inflate (one thread per placed candidate, gz_input_stream<true>).  gz[slot] carries a candidate from one pass to the next.
constexpr uint32_t kH2Gunzip = 2u;                                // H2Conn::pad0 bit: b2_h2_conn_set_gunzip
constexpr uint32_t kGzSkip = 0xffffffffu, kGzToHost = 0xfffffffeu, kGzToSize = 0xfffffffdu;
__global__ void k_h2_set_gunzip(H2Conn* conns, uint32_t conn, int enable) {
    if (enable) conns[conn].pad0 |= kH2Gunzip; else conns[conn].pad0 &= ~kH2Gunzip;
}
__device__ __forceinline__ bool h2gz_failed(const b2_h2_msg&) { return false; }
__device__ __forceinline__ bool h2gz_failed(const b2_h2_call& m) { return m.error_code != 0; }   // ProcessHttpResponse stopped before
// ... before its grpc-encoding check: with a valid prefix, ERESPONSE (2002) comes from that check itself
__device__ __forceinline__ bool h2gz_stopped_earlier(const b2_h2_msg&) { return false; }
__device__ __forceinline__ bool h2gz_stopped_earlier(const b2_h2_call& m) { return m.error_code != 0 && m.error_code != 2002; }
__device__ __forceinline__ bool h2gz_client(const b2_h2_msg&) { return false; }
__device__ __forceinline__ bool h2gz_client(const b2_h2_call&) { return true; }
// the compressed bytes: the gRPC message after its prefix, or the whole body
template <class M>
__device__ __forceinline__ const uint8_t* h2gz_src(const M& m, const uint8_t* bytes, const uint8_t* out, uint32_t& n) {
    const bool grpc = m.flags & B2_H2_FLAG_GRPC;
    n = grpc ? m.body_len - 5 : m.body_len;
    return ((m.flags & B2_H2_FLAG_BODY_IN_INPUT) ? bytes : out) + m.body_off + (grpc ? 5 : 0);
}
// The per-item bodies (run r, or descriptor slot t) of the four passes: the grid kernels below and k_h2_ring call them.
template <class M>
__device__ __forceinline__ void h2_gz_select_run(uint32_t r, const uint8_t* bytes, const b2_run* runs, const H2Conn* conns, const b2_h2_run_status* rs,
                                                 M* msgs, uint32_t per_run, const uint8_t* out, uint8_t* merge_scratch, uint32_t* gz) {
    const bool on = conns[(uint32_t)runs[r].socket_id].pad0 & kH2Gunzip;
    uint8_t* const scratch = merge_scratch + (size_t)r * kH2HdrBytes;
    for (uint32_t i = 0; i < rs[r].n_msgs; i++) {
        const uint32_t slot = r * per_run + i;
        gz[slot] = kGzSkip;
        if (!on) continue;
        M& m = msgs[slot];
        const uint8_t* recs = out + m.headers_off; uint32_t rl = m.headers_len;
        if (!h2gz_client(m)) {                                      // server records are raw: merge them as HttpHeader holds them
            uint32_t nh; int32_t sc = 200;
            rl = h2c_merge(recs, rl, scratch, nh, sc); recs = scratch;
        }
        const bool grpc = m.flags & B2_H2_FLAG_GRPC;
        const uint8_t* e; uint32_t el;
        bool has;
        if (grpc) {
            if (!(m.flags & B2_H2_FLAG_GRPC_PREFIX_OK) || !(m.flags & B2_H2_FLAG_GRPC_COMPRESSED)) continue;   // encoding stays NULL
            has = h2c_get(recs, rl, "grpc-encoding", e, el);
            if (!has) { if (!h2gz_stopped_earlier(m)) m.flags |= B2_H2_FLAG_NO_GRPC_ENCODING; continue; }
        } else {
            if (!h2gz_client(m) && m.body_len == 0) continue;      // ProcessHttpRequest: an empty body is not decoded
            has = h2c_get(recs, rl, "content-encoding", e, el);
        }
        if (!has || h2gz_failed(m) || !lit_eq(e, el, "gzip")) continue;   // *encoding == "gzip": the whole std::string
        uint32_t n;
        (void)h2gz_src(m, bytes, out, n);
        gz[slot] = n > kGzMaxIn ? kGzToHost : kGzToSize;
    }
}
template <class M>
__device__ __forceinline__ void h2_gz_size_one(uint32_t t, const uint8_t* bytes, const b2_h2_run_status* rs, const M* msgs, uint32_t per_run,
                                               const uint8_t* out, uint32_t* gz) {
    if (t % per_run >= rs[t / per_run].n_msgs || gz[t] != kGzToSize) return;
    uint32_t n;
    const uint8_t* src = h2gz_src(msgs[t], bytes, out, n);
    bool big = false;
    const uint32_t bound = gz_input_stream<false>(src, n, B2_COMPRESS_TYPE_GZIP, nullptr, kGzMaxOut, &big);
    gz[t] = big ? kGzToHost : bound;
}
template <class M>
__device__ __forceinline__ void h2_gz_place_run(uint32_t r, b2_h2_run_status* rs, M* msgs, uint32_t per_run, uint32_t region, uint32_t* gz) {
    uint32_t cur = region / 4 + rs[r].first_msg;                    // (the consume kernel reports its blob bytes there, a multiple of 16)
    for (uint32_t i = 0; i < rs[r].n_msgs; i++) {
        const uint32_t slot = r * per_run + i, g = gz[slot];
        if (g == kGzSkip) continue;
        if (g == kGzToHost || (unsigned long long)cur + g > region) { msgs[slot].flags |= B2_H2_FLAG_GUNZIP_HOST; gz[slot] = kGzSkip; continue; }
        msgs[slot].msg_off = r * region + cur;
        cur += (g + 15u) & ~15u;
    }
    rs[r].first_msg = cur - region / 4;                            // the strided copy-back brings the inflated bytes home
}
template <class M>
__device__ __forceinline__ void h2_gz_inflate_one(uint32_t t, const uint8_t* bytes, const b2_h2_run_status* rs, M* msgs, uint32_t per_run,
                                                  uint8_t* out, const uint32_t* gz) {
    if (t % per_run >= rs[t / per_run].n_msgs || gz[t] == kGzSkip) return;
    M& m = msgs[t];
    uint32_t n;
    const uint8_t* src = h2gz_src(m, bytes, out, n);
    bool big = false;
    m.msg_len = gz_input_stream<true>(src, n, B2_COMPRESS_TYPE_GZIP, out + m.msg_off, gz[t], &big);   // <= the bound: a failed check hands over less
    m.flags |= B2_H2_FLAG_GUNZIPPED;
}
template <class M>
__global__ void k_h2_gz_select(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, const H2Conn* conns, const b2_h2_run_status* rs,
                               M* msgs, uint32_t per_run, const uint8_t* out, uint8_t* merge_scratch, uint32_t* gz) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_runs) h2_gz_select_run(r, bytes, runs, conns, rs, msgs, per_run, out, merge_scratch, gz);
}
template <class M>
__global__ void k_h2_gz_size(const uint8_t* bytes, uint32_t n_runs, const b2_h2_run_status* rs, const M* msgs, uint32_t per_run,
                             const uint8_t* out, uint32_t* gz) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_runs * per_run) h2_gz_size_one(t, bytes, rs, msgs, per_run, out, gz);
}
template <class M>
__global__ void k_h2_gz_place(uint32_t n_runs, b2_h2_run_status* rs, M* msgs, uint32_t per_run, uint32_t region, uint32_t* gz) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_runs) h2_gz_place_run(r, rs, msgs, per_run, region, gz);
}
template <class M>
__global__ void k_h2_gz_inflate(const uint8_t* bytes, uint32_t n_runs, const b2_h2_run_status* rs, M* msgs, uint32_t per_run,
                                uint8_t* out, const uint32_t* gz) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_runs * per_run) h2_gz_inflate_one(t, bytes, rs, msgs, per_run, out, gz);
}

// ---------------------------------------------------------------------------------------------------------
// b2_h2_serve_batch: for gRPC calls of B2_HANDLER_ECHO methods, what follows the parse in brpc — ProcessHttpRequest's body checks
// (policy/http_rpc_protocol.cpp:1631-1689), EchoServiceImpl::Echo and SendHttpResponse (:852-1027) — over what h2_consume_run and
// the gunzip passes left on the device.  k_h2_serve (one thread per run: a connection's replies are ordered) decides every call,
// writes error texts and copied bodies into the run's out region and builds b2_h2_response records; k_h2_serve_scan and
// k_h2_serve_compact list them connection by connection for k_h2_pack, which frames them as for b2_h2_pack_responses;
// k_h2_serve_gather closes the gaps between a run's replies.
constexpr uint32_t kH2ServeCtMax = 256;                           // the content-type length b2_h2_pack_responses accepts
// The longest error text (Controller::SetFailed, controller.cpp:468-490): "[" identity "]" "[E1003]" then request_type_name and
// " needs to be created from a non-empty json, it has required fields." (67 bytes) = 1 + 63 + 1 + 7 + 95 + 67 = 234 bytes.
// PercentEncode makes each byte at most "%xx": 702 bytes of grpc-message, more than the 512 b2_h2_pack_responses takes from the host.
// k_h2_pack encodes it as a literal: the trailer holds grpc-status (at most 15 bytes) and grpc-message (1 + 1 + 12 + 3 length bytes +
// the value), its scratch name || value, and the connection's HPACK table an entry of name + value + 32 bytes.
struct H2ServeCfg { uint32_t n_methods, identity_len; char identity[64]; };   // of DevConfig: the registered methods, b2_set_server_identity
constexpr uint32_t kH2ServeTextMax = 1 + (sizeof(H2ServeCfg::identity) - 1) + 1 + 7 + (sizeof(DevMethod::request_type) - 1) + 67;
constexpr uint32_t kH2ServeMsgMax = 3 * kH2ServeTextMax;
static_assert(kH2ServeTextMax == 234 && kH2ServeMsgMax == 702, "the longest error text");
static_assert(15 + 17 + kH2ServeMsgMax <= kH2FragCap && 12 + kH2ServeMsgMax <= kH2FragCap, "grpc-message fits k_h2_pack's trailer and scratch");
static_assert(12 + kH2ServeMsgMax + 32 <= 4096, "grpc-message fits an HPACK table entry");
static_assert(1 + 2 + 3 + kH2ServeCtMax <= kH2FragCap && 12 + kH2ServeCtMax <= kH2FragCap, "content-type fits k_h2_pack's header block and scratch");
enum H2ServeWhy : uint32_t { kServeOk = 0, kServeEmpty, kServeBadPrefix, kServeNoEncoding, kServeParse };
// PercentEncode (grpc.cpp:121-141) of n bytes: only a-z A-Z - _ . ~ stay, everything else (digits too) is "%xx" in lowercase hex.
// Counts when p is null.
__device__ __forceinline__ uint32_t h2_pct(uint8_t* p, const uint8_t* s, uint32_t n) {
    uint32_t o = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t c = s[i];
        if ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '-' || c == '_' || c == '.' || c == '~') { if (p) p[o] = c; o++; }
        else { if (p) { p[o] = '%'; p[o + 1] = (uint8_t)"0123456789abcdef"[c >> 4]; p[o + 2] = (uint8_t)"0123456789abcdef"[c & 15]; } o += 3; }
    }
    return o;
}
__device__ __forceinline__ uint32_t h2_pct_lit(uint8_t* p, const char* lit) {
    uint32_t n = 0; while (lit[n]) n++;
    return h2_pct(p, (const uint8_t*)lit, n);
}
// the grpc-message of an EREQUEST reply: PercentEncode of SetFailed's text ("[ip:port]" when an identity is set, "[E1003]", the reason
// of ProcessHttpRequest :1637-1689); its length, and its bytes at p unless p is null
__device__ __noinline__ uint32_t h2_serve_error(uint8_t* p, const H2ServeCfg& C, const DevMethod& M, uint32_t why) {
    uint32_t o = 0;
    auto at = [&]() { return p ? p + o : nullptr; };
    if (C.identity_len) { o += h2_pct_lit(at(), "["); o += h2_pct(at(), (const uint8_t*)C.identity, C.identity_len); o += h2_pct_lit(at(), "]"); }
    o += h2_pct_lit(at(), "[E1003]");
    const uint8_t* rt = (const uint8_t*)M.request_type;
    switch (why) {
    case kServeEmpty: o += h2_pct(at(), rt, M.request_type_len); o += h2_pct_lit(at(), " needs to be created from a non-empty json, it has required fields."); break;
    case kServeBadPrefix: o += h2_pct_lit(at(), "Invalid gRPC request"); break;
    case kServeNoEncoding: o += h2_pct_lit(at(), "Fail to find header `grpc-encoding' in compressed gRPC request"); break;
    default: o += h2_pct_lit(at(), "Fail to parse http body as "); o += h2_pct(at(), rt, M.request_type_len); break;
    }
    return o;
}
// The records of run r go to resps / reply_offs[r * per_run ...], their count to spans[r].n_answered.  Reply i of the run gets
// h2_reply_bound bytes at reply_offs (16-byte aligned) in the run's reply_region bytes of the packed replies.
// k_h2_serve (a thread per run) and k_h2_ring call it.
__device__ __forceinline__ void h2_serve_run(uint32_t r, const uint8_t* bytes, const b2_run* runs, const DevMethod* methods, const H2ServeCfg& cfg,
                                             b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t per_run, uint8_t* out, uint32_t region,
                                             b2_h2_response* resps, uint32_t* reply_offs, uint32_t reply_region, b2_h2_reply_span* spans) {
    const uint32_t gbase = r * region;
    uint32_t cur = region / 4 + rs[r].first_msg;                    // behind the parse's and the gunzip passes' bytes (a multiple of 16)
    uint32_t rep = 0, k = 0;
    for (uint32_t i = 0; i < rs[r].n_msgs; i++) {
        b2_h2_msg& m = msgs[r * per_run + i];
        if (!(m.flags & B2_H2_FLAG_GRPC) || m.content_type != 2 /*HTTP_CONTENT_PROTO*/ || m.method_idx < 0 || (uint32_t)m.method_idx >= cfg.n_methods) continue;
        const DevMethod& M = methods[m.method_idx];
        if (M.handler != B2_HANDLER_ECHO || M.response_compress_type != B2_COMPRESS_TYPE_NONE) continue;
        uint32_t ct_off = 0, ct_len = 0;                            // SendHttpResponse answers with the request's content-type (:857-862)
        for (uint32_t q = 0; q < m.headers_len;) {
            const uint8_t* rec = out + m.headers_off + q;
            const uint32_t nl = rec[0] | ((uint32_t)rec[1] << 8), vl = rec[2] | ((uint32_t)rec[3] << 8);
            if (lit_eq(rec + 4, cstr_len(rec + 4, nl), "content-type")) { ct_off = m.headers_off + q + 4 + nl; ct_len = vl; }
            q += 4 + nl + vl;
        }
        if (ct_len > kH2ServeCtMax) continue;
        // ProcessHttpRequest (:1631-1689), in its order
        const uint8_t* src = (m.flags & B2_H2_FLAG_BODY_IN_INPUT) ? bytes : out;
        uint32_t why = kServeOk;
        Span msg; msg.off = 0; msg.len = 0;
        if (m.body_len == 0) why = kServeEmpty;                     // EchoRequest has a required field
        else if (!(m.flags & B2_H2_FLAG_GRPC_PREFIX_OK)) why = kServeBadPrefix;
        else if (m.flags & B2_H2_FLAG_GRPC_COMPRESSED) {
            if (m.flags & B2_H2_FLAG_NO_GRPC_ENCODING) why = kServeNoEncoding;
            else if (m.flags & B2_H2_FLAG_GUNZIPPED) src = out;     // the inflated bytes
            else continue;                                          // another encoding, or left to the host's zlib
        }
        if (why == kServeOk && !decode_echo_request(src + m.msg_off, m.msg_len, msg)) why = kServeParse;
        b2_h2_response R;
        R.conn = (uint32_t)runs[r].socket_id; R.stream_id = m.stream_id; R.status_code = 200;
        R.flags = B2_H2_RESP_GRPC | B2_H2_RESP_CT_IN_OUT; R.content_type_off = ct_off; R.content_type_len = ct_len;
        R.body_off = 0; R.body_len = 0; R.grpc_status = 0; R.grpc_message_off = 0; R.grpc_message_len = 0; R.reserved = 0;
        uint32_t put = 0;                                           // bytes the reply needs in out
        const uint32_t at = m.msg_off + msg.off, vn = varint_len(msg.len);
        if (why != kServeOk) {                                      // an empty body, the 5-byte prefix and the trailers (:937-959, :1008-1011)
            R.grpc_status = 3;                                      // ErrorCodeToGrpcStatus(EREQUEST), grpc.cpp:63-65
            put = R.grpc_message_len = h2_serve_error(nullptr, cfg, M, why);
        } else {                                                    // EchoResponse{message}: 0a varint(len) message
            R.body_len = 1 + vn + msg.len;
            // the request already holds that field when the tag is 0a and the length took exactly varint_len(len) bytes
            bool same = msg.off >= 1 + vn && src[at - vn - 1] == 0x0a;
            unsigned long long v = 0;
            for (uint32_t j = 0; same && j < vn; j++) {
                const uint8_t b = src[at - vn + j];
                same = (j + 1 < vn) == ((b & 0x80) != 0); v |= (unsigned long long)(b & 0x7f) << (7 * j);
            }
            if (same && v == msg.len) { R.body_off = at - vn - 1; R.flags |= src == bytes ? B2_H2_RESP_BODY_IN_INPUT : B2_H2_RESP_BODY_IN_OUT; }
            else put = R.body_len;
        }
        const uint64_t next = (rep + h2_reply_bound(R.body_len, ct_len, R.grpc_message_len) + 15) & ~15ull;
        if (next > reply_region) break;                             // the run's reply region is full: the rest is the host's
        if (put && (uint64_t)cur + put > region) continue;          // no room in out for this call's bytes
        if (why != kServeOk) { R.grpc_message_off = gbase + cur; (void)h2_serve_error(out + gbase + cur, cfg, M, why); }
        else if (put) {
            uint8_t* o = out + gbase + cur;
            *o++ = 0x0a; o = put_varint(o, msg.len);
            thread_copy(o, src + at, msg.len);
            R.body_off = gbase + cur; R.flags |= B2_H2_RESP_BODY_IN_OUT;
        }
        cur += (put + 15u) & ~15u;
        resps[r * per_run + k] = R; reply_offs[r * per_run + k] = r * reply_region + rep; k++;
        rep = (uint32_t)next;
        m.flags |= B2_H2_FLAG_ANSWERED; m.reserved = (uint32_t)R.grpc_status;
    }
    rs[r].first_msg = cur - region / 4;                             // the strided copy-back brings the texts and bodies home
    b2_h2_reply_span sp; sp.off = r * reply_region; sp.len = 0; sp.n_answered = k; sp.reserved = 0;
    spans[r] = sp;
}
__global__ void k_h2_serve(const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, const DevMethod* methods, const H2ServeCfg cfg,
                           b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t per_run, uint8_t* out, uint32_t region,
                           b2_h2_response* resps, uint32_t* reply_offs, uint32_t reply_region, b2_h2_reply_span* spans) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_runs) h2_serve_run(r, bytes, runs, methods, cfg, rs, msgs, per_run, out, region, resps, reply_offs, reply_region, spans);
}
// One warp: first[r] = the exclusive prefix of count(r) over the runs, first[n_runs] = the total.  Lane l sums a contiguous share.
template <class F>
__device__ __forceinline__ void h2_warp_scan_runs(uint32_t n_runs, uint32_t lane, F count, uint32_t* first) {
    const uint32_t per = (n_runs + 31) / 32;
    const uint32_t lo = min(lane * per, n_runs), hi = min(lo + per, n_runs);
    uint32_t sum = 0;
    for (uint32_t r = lo; r < hi; r++) sum += count(r);
    uint32_t incl = sum;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_sync(0xffffffffu, incl, lane >= d ? lane - d : lane);
        if (lane >= d) incl += v;
    }
    uint32_t at = incl - sum;
    for (uint32_t r = lo; r < hi; r++) { first[r] = at; at += count(r); }
    if (lane == 31) first[n_runs] = incl;
}
// One warp: group_first (k_h2_pack's list of connections, one per run, empty ones included) = the exclusive prefix of the answered counts
__global__ void k_h2_serve_scan(uint32_t n_runs, const b2_h2_reply_span* spans, uint32_t* group_first) {
    h2_warp_scan_runs(n_runs, threadIdx.x, [&](uint32_t r) { return spans[r].n_answered; }, group_first);
}
// one descriptor slot t: the record and reply offset move from per_run strides into that list
__device__ __forceinline__ void h2_serve_compact_one(uint32_t t, uint32_t per_run, const b2_h2_reply_span* spans, const uint32_t* group_first,
                                                     const b2_h2_response* strided, const uint32_t* strided_offs, b2_h2_response* resps, uint32_t* reply_offs) {
    const uint32_t r = t / per_run, k = t % per_run;
    if (k >= spans[r].n_answered) return;
    resps[group_first[r] + k] = strided[t]; reply_offs[group_first[r] + k] = strided_offs[t];
}
__global__ void k_h2_serve_compact(uint32_t n_runs, uint32_t per_run, const b2_h2_reply_span* spans, const uint32_t* group_first,
                                   const b2_h2_response* strided, const uint32_t* strided_offs, b2_h2_response* resps, uint32_t* reply_offs) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_runs * per_run) h2_serve_compact_one(t, per_run, spans, group_first, strided, strided_offs, resps, reply_offs);
}
// One warp per run: the replies k_h2_pack wrote at their reserved offsets move down to follow each other.  The move is forward inside
// the run's region: every 512-byte step is loaded whole before any of it is stored, and a step never stores past what it loaded.
__device__ __forceinline__ void h2_gather_run(uint32_t r, uint32_t lane, const uint32_t* group_first, const uint32_t* reply_offs,
                                              const uint32_t* reply_lens, uint8_t* replies, b2_h2_reply_span* spans) {
    const uint32_t start = spans[r].off;
    uint32_t dst = start;
    for (uint32_t i = group_first[r]; i < group_first[r + 1]; i++) {
        const uint32_t src = reply_offs[i], n = reply_lens[i];
        if (src != dst) {
            for (uint32_t s = 0; s < n; s += 512) {
                const uint32_t o = s + 16 * lane;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (o < n) v = *reinterpret_cast<const uint4*>(replies + src + o);     // (src is 16-byte aligned)
                __syncwarp();
#pragma unroll
                for (uint32_t j = 0; j < 16; j++)
                    if (o + j < n) replies[dst + o + j] = (uint8_t)((j < 4 ? v.x : j < 8 ? v.y : j < 12 ? v.z : v.w) >> (8 * (j & 3)));
                __syncwarp();
            }
        }
        dst += n;
    }
    if (lane == 0) spans[r].len = dst - start;
}
__global__ void __launch_bounds__(kH2PackWarps * 32) k_h2_serve_gather(uint32_t n_runs, const uint32_t* group_first, const uint32_t* reply_offs,
                                                                       const uint32_t* reply_lens, uint8_t* replies, b2_h2_reply_span* spans) {
    const uint32_t lane = threadIdx.x & 31, r = blockIdx.x * kH2PackWarps + (threadIdx.x >> 5);
    if (r < n_runs) h2_gather_run(r, lane, group_first, reply_offs, reply_lens, replies, spans);
}

#if defined(B2_KERNELS_RING)
// ---------------------------------------------------------------------------------------------------------
// The block phases k_h2_ring and k_h2_client_ring share.  The four gunzip passes over the ticket's parse (the whole CTA, __syncthreads()
// where the batch call has kernel boundaries).
template <class M>
__device__ __forceinline__ void h2_ring_gunzip(uint32_t n_runs, uint32_t per_run, uint32_t region, const uint8_t* bytes, const b2_run* runs,
                                               const H2Conn* conns, b2_h2_run_status* rs, M* msgs, uint8_t* out, uint8_t* merge, uint32_t* gz) {
    const uint32_t tid = threadIdx.x, n_slots = n_runs * per_run;
    for (uint32_t r = tid; r < n_runs; r += kSmallThreads) h2_gz_select_run(r, bytes, runs, conns, rs, msgs, per_run, out, merge, gz);
    __syncthreads();
    for (uint32_t i = tid; i < n_slots; i += kSmallThreads) h2_gz_size_one(i, bytes, rs, msgs, per_run, out, gz);
    __syncthreads();
    for (uint32_t r = tid; r < n_runs; r += kSmallThreads) h2_gz_place_run(r, rs, msgs, per_run, region, gz);
    __syncthreads();
    for (uint32_t i = tid; i < n_slots; i += kSmallThreads) h2_gz_inflate_one(i, bytes, rs, msgs, per_run, out, gz);
    __syncthreads();
}
// The push of run r, by one warp: its descriptors into the list at first[r] (the batch call compacts them on the host), its control
// bytes and blob (whose length the status reports in first_msg) at the offsets the batch call uses, then the status with first_msg =
// the list index.
template <class M>
__device__ __forceinline__ void h2_ring_push_run(uint32_t r, uint32_t lane, uint8_t* slot, uint32_t off_rs, uint32_t off_descs, uint32_t off_out,
                                                 const b2_h2_run_status* rs, const M* descs, uint32_t per_run, const uint8_t* out, uint32_t region,
                                                 const uint32_t* first) {
    b2_h2_run_status st = rs[r];
    const uint32_t f = first[r], base = r * region;
    ring_push(slot + off_descs + (size_t)f * sizeof(M), reinterpret_cast<const uint8_t*>(descs + (size_t)r * per_run), st.n_msgs * (uint32_t)sizeof(M), lane, 32);
    ring_push(slot + off_out + base, out + base, st.ctrl_len, lane, 32);
    ring_push(slot + off_out + base + region / 4, out + base + region / 4, st.first_msg, lane, 32);
    if (lane == 0) { st.first_msg = f; reinterpret_cast<b2_h2_run_status*>(slot + off_rs)[r] = st; }
}
// k_h2_ring: b2_h2_serve_batch on the latency path (b2_h2_ring_*).  One resident CTA, fed through the same submit ring as k_ring
// (the ticket loop ring_serve and ring_push of b2_kernels.cuh): per ticket the passes of the batch call, as block phases with
// __syncthreads() where the batch call has kernel boundaries, on the same device scratch, then only the used parts are pushed into the
// ticket's slot.  H2Conn, HpackState and the stream pool are read through L1: every call that writes them from another kernel retires
// this one first (ring_halt), so a launch boundary lies between their writes and this CTA's loads.
// A turn (b2_h2_ring_turn_*) also carries the replies the host produced: after the served replies, b2_h2_pack_responses over them as
// one more block phase, so that they take the encoder table and windows the served replies left.  Their block (records, the offsets the
// host placed, group_first) is pulled into scratch of its own (turn), which also holds their lengths and frames; only out_len bytes of
// each frame are pushed.  The phase is k_h2_ring<true>'s (b2_h2_ring_turn_enable): k_h2_ring<false> is the kernel without it, so that
// contexts without turns keep its registers, stack and spills as they were.
struct H2RingArgs { uint32_t per_run, region, reply_region, gunzip, n_resps, n_groups, pad[2]; };   // per ticket, from the host, at the slot's off_args
// the host-reply block of a turn: n records, their placed offsets, then group_first (n_groups + 1 words); all parts 16-byte aligned
B2_HD uint32_t h2r_turn_offs_off(uint32_t n) { return n * (uint32_t)sizeof(b2_h2_response); }
B2_HD uint32_t h2r_turn_first_off(uint32_t n) { return h2r_turn_offs_off(n) + ((n * 4 + 15u) & ~15u); }
B2_HD uint32_t h2r_turn_block(uint32_t n, uint32_t n_groups) { return h2r_turn_first_off(n) + (((n_groups + 1) * 4 + 15u) & ~15u); }
struct H2RingDev {
    uint32_t off_args, off_rs, off_msgs, off_spans, off_out, off_replies;  // the slot's parts behind RingSlotHdr (runs, staged input: RingDev)
    H2Conn* conns; HpackState* hps; const DevMethod* methods; uint32_t n_methods; H2ServeCfg cfg; H2Pool pool;
    // the scratch of b2_h2_serve_batch: the run statuses, per_run-strided descriptors, the out regions, the gunzip merge scratch, gz words
    // (then the reply lengths), the strided records and their offsets, the list k_h2_pack reads and its offsets, group_first (then the
    // first list index of every run's messages), the spans and the replies
    b2_h2_run_status* rs; b2_h2_msg* msgs; uint8_t* out; uint8_t* merge; uint32_t* gz;
    b2_h2_response* strided; uint32_t* strided_offs; b2_h2_response* list; uint32_t* list_offs; uint32_t* first;
    b2_h2_reply_span* spans; uint8_t* replies;
};
// k_h2_ring<true>'s own parts (a parameter of their own, so that k_h2_ring<false> keeps H2RingDev's size and stack): the slot's
// host-reply block, lengths and frames, and the device scratch they are pulled into and packed in
struct H2TurnDev {
    uint32_t off_resps, off_resp_lens, off_resp_out;
    uint8_t* turn; uint32_t* turn_lens; uint8_t* turn_out;
};
constexpr uint32_t kH2RingSmem = kSmallWarps * 3 * kH2FragCap;          // k_h2_pack's scratch for each warp
template <bool kReplies>
__global__ void __launch_bounds__(kSmallThreads, 1) k_h2_ring(RingDev R, H2RingDev H, H2TurnDev Q) {
    extern __shared__ __align__(16) uint8_t h2_ring_raw[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint8_t* bytes = R.d_bytes;
    const b2_run* runs = reinterpret_cast<const b2_run*>(R.d_meta);
    ring_serve<H2RingArgs>(R, H.off_args, [] {}, [&](uint8_t* slot, const RingSlotHdr& s_hdr, const H2RingArgs& s_args, unsigned long long (&t)[4]) __attribute__((always_inline)) {
        const uint32_t n_runs = s_hdr.n_runs, per_run = s_args.per_run, region = s_args.region, reply_region = s_args.reply_region, n_slots = n_runs * per_run;
        if constexpr (kReplies) {
            if (s_args.n_resps) {   // the host-reply block, while the serve passes below run (they never touch it)
                const uint4* src = reinterpret_cast<const uint4*>(slot + Q.off_resps);
                uint4* dst = reinterpret_cast<uint4*>(Q.turn);
                for (uint32_t k = tid; k < h2r_turn_block(s_args.n_resps, s_args.n_groups) / 16u; k += kSmallThreads) dst[k] = src[k];
            }
        }
        for (uint32_t r = tid; r < n_runs; r += kSmallThreads)
            h2_consume_run<false>(r, bytes, runs, H.conns, H.hps, H.methods, H.n_methods, H.rs, H.msgs, per_run, H.out, region, H.pool);
        __syncthreads();
        if (s_args.gunzip) h2_ring_gunzip(n_runs, per_run, region, bytes, runs, H.conns, H.rs, H.msgs, H.out, H.merge, H.gz);   // a run's connection opted in
        for (uint32_t r = tid; r < n_runs; r += kSmallThreads)
            h2_serve_run(r, bytes, runs, H.methods, H.cfg, H.rs, H.msgs, per_run, H.out, region, H.strided, H.strided_offs, reply_region, H.spans);
        __syncthreads();
        if (wid == 0) h2_warp_scan_runs(n_runs, lane, [&](uint32_t r) { return H.spans[r].n_answered; }, H.first);
        __syncthreads();
        for (uint32_t i = tid; i < n_slots; i += kSmallThreads) h2_serve_compact_one(i, per_run, H.spans, H.first, H.strided, H.strided_offs, H.list, H.list_offs);
        __syncthreads();
        for (uint32_t g = wid; g < n_runs; g += kSmallWarps)
            h2_pack_group(g, lane, h2_ring_raw + wid * 3 * kH2FragCap, H.out, bytes, H.out, H.list, H.first, H.conns, H.replies, H.list_offs, H.gz);
        __syncthreads();
        for (uint32_t r = wid; r < n_runs; r += kSmallWarps) h2_gather_run(r, lane, H.first, H.list_offs, H.gz, H.replies, H.spans);
        __syncthreads();
        if constexpr (kReplies) {
            if (s_args.n_resps) {   // the host's replies, framed against the encoder tables and windows the served replies just moved
                const uint32_t n_resps = s_args.n_resps;
                for (uint32_t g = wid; g < s_args.n_groups; g += kSmallWarps)
                    h2_pack_group(g, lane, h2_ring_raw + wid * 3 * kH2FragCap, bytes, nullptr, nullptr, reinterpret_cast<const b2_h2_response*>(Q.turn),
                                  reinterpret_cast<const uint32_t*>(Q.turn + h2r_turn_first_off(n_resps)), H.conns, Q.turn_out,
                                  reinterpret_cast<const uint32_t*>(Q.turn + h2r_turn_offs_off(n_resps)), Q.turn_lens);
                __syncthreads();
            }
        }
        if (tid == 0) t[3] = globaltimer_ns();                          // replies packed
        // the descriptors become one list in run order (the batch call compacts them on the host): first[r] = run r's first list index
        if (wid == 0) h2_warp_scan_runs(n_runs, lane, [&](uint32_t r) { return H.rs[r].n_msgs; }, H.first);
        __syncthreads();
        // push, a warp per run: h2_ring_push_run, then its replies and span
        for (uint32_t r = wid; r < n_runs; r += kSmallWarps) {
            const b2_h2_reply_span sp = H.spans[r];
            h2_ring_push_run(r, lane, slot, H.off_rs, H.off_msgs, H.off_out, H.rs, H.msgs, per_run, H.out, region, H.first);
            ring_push(slot + H.off_replies + sp.off, H.replies + sp.off, sp.len, lane, 32);
            if (lane == 0) reinterpret_cast<b2_h2_reply_span*>(slot + H.off_spans)[r] = sp;
        }
        if constexpr (kReplies) {
            if (s_args.n_resps) {   // the host replies' lengths, then a warp per reply its frames
                const uint32_t n_resps = s_args.n_resps;
                const uint32_t* offs = reinterpret_cast<const uint32_t*>(Q.turn + h2r_turn_offs_off(n_resps));
                ring_push(slot + Q.off_resp_lens, reinterpret_cast<const uint8_t*>(Q.turn_lens), n_resps * 4u, tid, kSmallThreads);
                for (uint32_t i = wid; i < n_resps; i += kSmallWarps) ring_push(slot + Q.off_resp_out + offs[i], Q.turn_out + offs[i], __ldcg(Q.turn_lens + i), lane, 32);
            }
        }
        return false;
    });
}

// ---------------------------------------------------------------------------------------------------------
// k_h2_client_ring: one turn of a client's event loop on the latency path (b2_h2_client_ring_*): b2_h2_client_process_batch over the
// ticket's runs, then b2_h2_pack_requests over its requests, as block phases on the same device scratch, so that what the runs change
// (SETTINGS, WINDOW_UPDATE, GOAWAY, ended calls) governs the requests of the same ticket.  The requests, their placed results and
// group_first are pulled from the slot into scratch the parse does not use, and their fields index the pulled input; frames go to
// the offsets the host placed, and only out_len bytes of each are pushed.  Connection state is read through L1, as in k_h2_ring.
struct H2ClientRingArgs { uint32_t per_run, region, gunzip, n_reqs, n_groups, pad[3]; };   // per ticket, from the host, at the slot's off_args
struct H2ClientRingDev {
    // the slot's parts behind RingSlotHdr (runs, staged input: RingDev); off_reqs: [requests | placed results | group_first] of the ticket
    uint32_t off_args, off_reqs, off_rs, off_calls, off_out, off_req_res, off_req_out;
    H2Conn* conns; HpackState* hps; H2Pool pool;
    // the scratch of b2_h2_client_process_batch (statuses, per_run-strided calls, out regions, gunzip merge scratch and words, then the
    // first list index of every run's calls), the pulled request block, and the frames of b2_h2_pack_requests
    b2_h2_run_status* rs; b2_h2_call* calls; uint8_t* out; uint8_t* merge; uint32_t* gz; uint32_t* first;
    uint8_t* reqs; uint8_t* req_out;
};
// the request block of a ticket: n requests, their results (out_off placed), then group_first (n_groups + 1 words); all parts 16-byte aligned
B2_HD uint32_t h2c_ring_res_off(uint32_t n) { return n * (uint32_t)sizeof(b2_h2_request); }
B2_HD uint32_t h2c_ring_first_off(uint32_t n) { return h2c_ring_res_off(n) + n * (uint32_t)sizeof(b2_h2_request_result); }
B2_HD uint32_t h2c_ring_block(uint32_t n, uint32_t n_groups) { return h2c_ring_first_off(n) + (((n_groups + 1) * 4 + 15u) & ~15u); }
constexpr uint32_t kH2ClientRingSmem = kSmallWarps * 2 * kH2ReqFragCap;  // k_h2_pack_req's scratch for each warp
__global__ void __launch_bounds__(kSmallThreads, 1) k_h2_client_ring(RingDev R, H2ClientRingDev H) {
    extern __shared__ __align__(16) uint8_t h2c_ring_raw[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint8_t* bytes = R.d_bytes;
    const b2_run* runs = reinterpret_cast<const b2_run*>(R.d_meta);
    ring_serve<H2ClientRingArgs>(R, H.off_args, [] {}, [&](uint8_t* slot, const RingSlotHdr& s_hdr, const H2ClientRingArgs& s_args, unsigned long long (&t)[4]) __attribute__((always_inline)) {
        const uint32_t n_runs = s_hdr.n_runs, per_run = s_args.per_run, region = s_args.region, n_reqs = s_args.n_reqs, n_groups = s_args.n_groups;
        const b2_h2_request* reqs = reinterpret_cast<const b2_h2_request*>(H.reqs);
        b2_h2_request_result* res = reinterpret_cast<b2_h2_request_result*>(H.reqs + h2c_ring_res_off(n_reqs));
        const uint32_t* group_first = reinterpret_cast<const uint32_t*>(H.reqs + h2c_ring_first_off(n_reqs));
        {   // the request block, while the parse below has not yet run (nothing reads it before the pack phase)
            const uint4* src = reinterpret_cast<const uint4*>(slot + H.off_reqs);
            uint4* dst = reinterpret_cast<uint4*>(H.reqs);
            for (uint32_t k = tid; k < h2c_ring_block(n_reqs, n_groups) / 16u; k += kSmallThreads) dst[k] = src[k];
        }
        for (uint32_t r = tid; r < n_runs; r += kSmallThreads)
            h2_consume_run<true>(r, bytes, runs, H.conns, H.hps, nullptr, 0, H.rs, H.calls, per_run, H.out, region, H.pool);
        __syncthreads();
        if (s_args.gunzip) h2_ring_gunzip(n_runs, per_run, region, bytes, runs, H.conns, H.rs, H.calls, H.out, H.merge, H.gz);   // a run's connection opted in
        for (uint32_t g = wid; g < n_groups; g += kSmallWarps)
            h2_pack_req_group(g, lane, h2c_ring_raw + wid * 2 * kH2ReqFragCap, bytes, reqs, group_first, H.conns, H.req_out, res, H.pool);
        __syncthreads();
        if (tid == 0) t[3] = globaltimer_ns();                          // requests packed
        if (wid == 0) h2_warp_scan_runs(n_runs, lane, [&](uint32_t r) { return H.rs[r].n_msgs; }, H.first);
        __syncthreads();
        // push: a warp per run (h2_ring_push_run), the request results, then a warp per request its frames
        for (uint32_t r = wid; r < n_runs; r += kSmallWarps)
            h2_ring_push_run(r, lane, slot, H.off_rs, H.off_calls, H.off_out, H.rs, H.calls, per_run, H.out, region, H.first);
        ring_push(slot + H.off_req_res, reinterpret_cast<const uint8_t*>(res), n_reqs * (uint32_t)sizeof(b2_h2_request_result), tid, kSmallThreads);
        for (uint32_t i = wid; i < n_reqs; i += kSmallWarps) {
            const b2_h2_request_result q = res[i];
            ring_push(slot + H.off_req_out + q.out_off, H.req_out + q.out_off, q.out_len, lane, 32);
        }
        return false;
    });
}
#endif
#endif
}  // namespace b2
