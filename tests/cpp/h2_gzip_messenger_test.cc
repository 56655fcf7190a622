// C++ test of b2::GpuH2Messenger with SetGunzip(true): gRPC echo requests that arrive gzip-compressed (grpc-encoding: gzip, prefix flag 1)
// are inflated on the device and echoed from `out` through B2_H2_RESP_BODY_IN_OUT, uncompressed; uncompressed requests on the same
// connections are echoed as before; a compressed request the device cannot inflate for brpc (no grpc-encoding) goes to the host callback.
// Every byte written back is compared with the oracle: the C oracle's parse and reply framing, the request inflated by its GzipInputStream.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../brpc_b200/host/h2_messenger.h"
#include "../../oracle/b2_oracle.h"

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #c); exit(1); } } while (0)

static std::string h2_frame(int type, int flags, uint32_t sid, const std::string& payload) {
    std::string f; const uint32_t n = (uint32_t)payload.size();
    f.push_back((char)(n >> 16)); f.push_back((char)(n >> 8)); f.push_back((char)n); f.push_back((char)type); f.push_back((char)flags);
    f.push_back((char)(sid >> 24)); f.push_back((char)(sid >> 16)); f.push_back((char)(sid >> 8)); f.push_back((char)sid);
    return f + payload;
}
static std::string hp_lit(const std::string& n, const std::string& v) {      // literal header field without indexing, new name (RFC 7541 6.2.2)
    std::string o; o.push_back(0); o.push_back((char)n.size()); o += n; o.push_back((char)v.size()); o += v; return o;
}
static uint32_t crc32_ieee(const std::string& s) {
    uint32_t c = 0xffffffffu;
    for (unsigned char b : s) { c ^= b; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xedb88320u & (0u - (c & 1u))); }
    return ~c;
}
static void put_le32(std::string& o, uint32_t v) { for (int i = 0; i < 4; i++) o.push_back((char)(v >> (8 * i))); }
// RFC 1952 member of stored DEFLATE blocks (RFC 1951 3.2.4), at most 65535 bytes each
static std::string gzip_stored(const std::string& data) {
    std::string o("\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff", 10);
    size_t at = 0;
    do {
        const size_t n = std::min<size_t>(65535, data.size() - at); const bool last = at + n == data.size();
        o.push_back(last ? 1 : 0); o.push_back((char)n); o.push_back((char)(n >> 8)); o.push_back((char)~n); o.push_back((char)(~n >> 8));
        o += data.substr(at, n); at += n;
    } while (at < data.size());
    put_le32(o, crc32_ieee(data)); put_le32(o, (uint32_t)data.size());
    return o;
}
static std::string grpc_body(const std::string& msg, bool compressed) {
    std::string b; b.push_back(compressed ? 1 : 0);
    b.push_back((char)(msg.size() >> 24)); b.push_back((char)(msg.size() >> 16)); b.push_back((char)(msg.size() >> 8)); b.push_back((char)msg.size());
    return b + msg;
}
static int g_host = 0;
static void HostProcess(b2::InputMessageBase* base) {
    b2::H2Message* m = static_cast<b2::H2Message*>(base);
    CHECK((m->desc.flags & B2_H2_FLAG_GRPC_COMPRESSED) && (m->desc.flags & B2_H2_FLAG_NO_GRPC_ENCODING));
    g_host++; delete m;
}

int main() {
    b2_options opt; memset(&opt, 0, sizeof opt);
    opt.device = 0; opt.max_batch_bytes = 8 << 20; opt.max_msgs = 1 << 14; opt.max_runs = 64; opt.max_resp_bytes = 32 << 20;
    b2::GpuH2Messenger messenger(opt, 32u << 20, 64, 32, 69632);
    b2_method echo = { "example.EchoService", "EchoService", "Echo", "example.EchoRequest", B2_HANDLER_ECHO, 1, 0, 0 };
    CHECK(messenger.AddMethod(echo) == 0);
    messenger.SetHostProcess(HostProcess);
    messenger.SetGunzip(true);
    const int kConns = 4, kCalls = 16;
    std::vector<std::string> streams(kConns);
    int n_compressed = 0;
    for (int c = 0; c < kConns; c++) {
        std::string& st = streams[c];
        st = "PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n"; st += h2_frame(4, 0, 0, "");
        for (int k = 0; k < kCalls; k++) {
            const uint32_t sid = 1 + 2 * k;
            const bool gz = k % 4 != 0, no_encoding = c == 1 && k == 5;
            std::string msg(7 + 53 * k + (k == 9 ? 30000 : 0), (char)('a' + (k + c) % 26));
            std::string hb = hp_lit(":method", "POST") + hp_lit(":scheme", "http") + hp_lit(":path", "/example.EchoService/Echo") +
                             hp_lit("content-type", "application/grpc") + hp_lit("te", "trailers") +
                             (no_encoding ? std::string() : hp_lit("grpc-encoding", "gzip"));     // the small plain ones carry it too, as grpcio sends
            const std::string body = grpc_body(gz ? gzip_stored(msg) : msg, gz);
            n_compressed += gz && !no_encoding;
            st += h2_frame(1, 0x4, sid, hb);
            if (k % 3 == 1) { st += h2_frame(0, 0, sid, body.substr(0, 9)); st += h2_frame(0, 0x1, sid, body.substr(9)); }   // the body assembled in the slot
            else if (body.size() > 16000) { st += h2_frame(0, 0, sid, body.substr(0, 16000)); st += h2_frame(0, 0x1, sid, body.substr(16000)); }
            else st += h2_frame(0, 0x1, sid, body);
        }
    }
    std::vector<b2::Socket*> socks; std::vector<size_t> pos(kConns, 0);
    std::vector<orc_h2_conn*> oc(kConns); std::vector<std::string> obuf(kConns), expect(kConns);
    for (int c = 0; c < kConns; c++) { socks.push_back(messenger.AddConnection(900 + c)); CHECK(socks.back()); oc[c] = orc_h2_conn_new(); }
    orc_config cfg; memset(&cfg, 0, sizeof cfg); b2_method ms[1] = { echo }; cfg.methods = ms; cfg.n_methods = 1;
    unsigned seed = 4242; int rounds = 0, total = 0, n_echo = 0;
    std::vector<b2_h2_msg> om(256); std::vector<uint8_t> octrl(1 << 16), oblob(1 << 21), opack(1 << 18);
    for (bool more = true; more; rounds++) {
        more = false;
        for (int c = 0; c < kConns; c++) {
            seed = seed * 1103515245u + 12345u;
            const size_t n = std::min(streams[c].size() - pos[c], (size_t)(seed >> 16) % 7000);
            socks[c]->_read_buf.append(streams[c].data() + pos[c], n); obuf[c].append(streams[c].data() + pos[c], n); pos[c] += n;
            if (pos[c] < streams[c].size()) more = true;
        }
        const int n = messenger.ProcessNewMessages(socks);
        CHECK(n >= 0); total += n;
        for (int c = 0; c < kConns; c++) {                       // the same round through the oracle
            if (obuf[c].empty()) continue;
            uint32_t cons = 0, nm = 0, cl = 0, bl = 0, mfs = 0, sws = 0;
            const uint32_t err = orc_h2_consume(oc[c], &cfg, (const uint8_t*)obuf[c].data(), (uint32_t)obuf[c].size(), &cons, om.data(), 256, &nm,
                                                octrl.data(), (uint32_t)octrl.size(), &cl, oblob.data(), (uint32_t)oblob.size(), &bl, &mfs, &sws);
            CHECK(err == B2_PARSE_ERROR_NOT_ENOUGH_DATA);
            expect[c].append((const char*)octrl.data(), cl);
            for (uint32_t k = 0; k < nm; k++) {
                std::string ct, enc; bool has_enc = false;
                for (uint32_t q = 0; q < om[k].headers_len;) {
                    const uint8_t* p = oblob.data() + om[k].headers_off + q; const uint32_t nl = p[0] | (p[1] << 8), vl = p[2] | (p[3] << 8);
                    if (nl == 12 && memcmp(p + 4, "content-type", 12) == 0) ct.assign((const char*)p + 4 + nl, vl);
                    if (nl == 13 && memcmp(p + 4, "grpc-encoding", 13) == 0) { enc.assign((const char*)p + 4 + nl, vl); has_enc = true; }
                    q += 4 + nl + vl;
                }
                std::string msg((const char*)oblob.data() + om[k].msg_off, om[k].msg_len);
                if (om[k].flags & B2_H2_FLAG_GRPC_COMPRESSED) {
                    if (!has_enc) continue;                      // EREQUEST: the host callback's business
                    CHECK(enc == "gzip");
                    uint8_t* inflated = nullptr; size_t il = 0;
                    CHECK(orc_gzip_input_stream((const uint8_t*)msg.data(), msg.size(), B2_COMPRESS_TYPE_GZIP, &inflated, &il) == 0);
                    msg.assign((const char*)inflated, il); orc_free(inflated);
                }
                std::string blob = ct + msg;
                b2_h2_response r; memset(&r, 0, sizeof r);
                r.stream_id = om[k].stream_id; r.status_code = 200; r.flags = B2_H2_RESP_GRPC; r.content_type_len = (uint32_t)ct.size();
                r.body_off = (uint32_t)ct.size(); r.body_len = (uint32_t)msg.size();
                const uint32_t pn = orc_h2_pack_response(oc[c], &r, (const uint8_t*)blob.data(), opack.data());
                expect[c].append((const char*)opack.data(), pn); n_echo++;
            }
            obuf[c].erase(0, cons);
        }
    }
    for (int c = 0; c < kConns; c++) {
        CHECK(!socks[c]->Failed() && socks[c]->_read_buf.length() == obuf[c].size());
        CHECK(socks[c]->_write_buf.to_string() == expect[c]);
        orc_h2_conn_free(oc[c]);
    }
    CHECK(total == kConns * kCalls && g_host == 1 && n_echo == kConns * kCalls - 1 && n_compressed > 40);
    printf("h2 gunzip messenger ok: %d connections, %d gRPC calls (%d gzip-compressed) in %d rounds, every written byte identical to the oracle, %d host-handled\n",
           kConns, total, n_compressed, rounds, g_host);
    return 0;
}
