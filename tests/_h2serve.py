"""Test oracle of b2_h2_serve_batch: what brpc does after ParseH2Message for a gRPC call of an echo method, with the device's placement,
so that the answered set, the spans and every reply byte compare.

  - which calls: gRPC, content type HTTP_CONTENT_PROTO, a B2_HANDLER_ECHO method without response compression, a content-type value of
    at most 256 bytes (the limit b2_h2_pack_responses keeps); everything else is the host's;
  - ProcessHttpRequest (src/brpc/policy/http_rpc_protocol.cpp:1631-1689), in its order: an empty body cannot make an EchoRequest, which
    has a required field (:1637-1643); RemoveGrpcPrefix (:1650-1655); a compressed message needs grpc-encoding (:1656-1664), is inflated
    when it is "gzip" (the gunzip step of _h2gzip: B2_H2_FLAG_GUNZIPPED) and is otherwise not answered; ParsePbFromIOBuf (:1684-1689),
    the C oracle's EchoRequest parser;
  - EchoServiceImpl::Echo: EchoResponse{message} = 0a varint(len) message;
  - Controller::SetFailed (src/brpc/controller.cpp:468-490): "[ip:port]" (AppendServerIdentiy), "[E1003]", the reason;
  - SendHttpResponse (:852-1027) for gRPC: :status 200, the request's content-type (:857-862), on failure an empty message (:937-940)
    behind AddGrpcPrefix (:1008-1011); H2UnsentResponse (src/brpc/policy/http2_rpc_protocol.cpp:1640-1650): grpc-status
    ErrorCodeToGrpcStatus (src/brpc/grpc.cpp:54-81), grpc-message PercentEncode (grpc.cpp:121-141) of the error text; the framing is
    the C oracle's pack_response (AppendAndDestroySelf + PackH2Message);
  - the device's placement: error texts and bodies that are not already in the request go 16-byte aligned behind the parse's and the
    gunzip's bytes of the run's out region (a call that does not fit is not answered); every answered call reserves
    h2_reply_bound bytes, 16-byte aligned, in the run's reply region, and the first that does not fit ends the run's answering."""
import _h2gzip as G
import _oracle as O
from _h2client_loop import records

F_GRPC, F_PREFIX_OK, F_COMPRESSED, F_BODY_IN_INPUT = 1, 2, 4, 16
F_GUNZIPPED, F_NO_GRPC_ENCODING, F_ANSWERED = G.F_GUNZIPPED, G.F_NO_GRPC_ENCODING, 512
HTTP_CONTENT_PROTO, HANDLER_ECHO, EREQUEST, GRPC_INVALIDARGUMENT, CT_MAX = 2, 1, 1003, 3, 256
a16 = G.a16


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def percent_encode(b):
    """PercentEncode (grpc.cpp:121-141): a-z A-Z - _ . ~ stay, every other byte is %xx in lowercase hex (digits included)"""
    return b"".join(bytes([c]) if (97 <= c <= 122 or 65 <= c <= 90 or c in b"-_.~") else b"%%%02x" % c for c in b)


def error_text(identity, reason):
    """Controller::SetFailed(EREQUEST, ...) on a server call (nretry 0): AppendServerIdentiy, "[E1003]", the reason"""
    return (b"[" + identity + b"]" if identity else b"") + b"[E%d]" % EREQUEST + reason


def reason_empty(request_type):
    return request_type + b" needs to be created from a non-empty json, it has required fields."


REASON_PREFIX = b"Invalid gRPC request"
REASON_NO_ENCODING = b"Fail to find header `grpc-encoding' in compressed gRPC request"


def reason_parse(request_type):
    return b"Fail to parse http body as " + request_type


def reply_bound(body_len, ct_len, gm_len):
    """h2_reply_bound: what b2_h2_pack_responses and b2_h2_serve_batch reserve for one reply"""
    data = body_len + 5
    return data + 9 * (data // 16384 + 4) + 2 * (ct_len + gm_len + 64) + 13 + 16


def content_type(hdr):
    """the last content-type header among the raw records (HttpHeader::set_content_type keeps the last one)"""
    ct = None
    for n, v in records(hdr):
        if n.split(b"\0")[0] == b"content-type":
            ct = v
    return ct


def decide(flags, ctype, method, ct, body, msg, identity):
    """One call: None when it is the host's, else dict(status, gm = grpc-message, body = the response message, copy = whether the body
    must be written into out)"""
    if not flags & F_GRPC or ctype != HTTP_CONTENT_PROTO or method is None:
        return None
    if method["handler"] != HANDLER_ECHO or method["response_compress_type"] != 0 or ct is None or len(ct) > CT_MAX:
        return None
    rt = method["request_type_name"]
    why = None
    if not body:
        why = reason_empty(rt)
    elif not flags & F_PREFIX_OK:
        why = REASON_PREFIX
    elif flags & F_COMPRESSED and flags & F_NO_GRPC_ENCODING:
        why = REASON_NO_ENCODING
    elif flags & F_COMPRESSED and not flags & F_GUNZIPPED:
        return None
    else:
        ok, (off, n) = O.parse_echo_request(msg)
        if not ok:
            why = reason_parse(rt)
        else:
            head = b"\x0a" + varint(n)
            resp = head + msg[off:off + n]
            return dict(status=0, gm=b"", body=resp, ct=ct, copy=not (off >= len(head) and msg[off - len(head):off] == head))
    return dict(status=GRPC_INVALIDARGUMENT, gm=percent_encode(error_text(identity, why)), body=b"", ct=ct, copy=True)


def place(decisions, region, out_used, reply_region):
    """k_h2_serve's placement over one run: [answered?], the out bytes used behind region / 4 afterwards, the reserved reply offsets"""
    cur = region // 4 + out_used; rep = 0; got = []; offs = []
    for d in decisions:
        if d is None:
            got.append(False); continue
        nxt = a16(rep + reply_bound(len(d["body"]), len(d["ct"]), len(d["gm"])))
        if nxt > reply_region:
            got += [False] * (len(decisions) - len(got))
            break
        put = (len(d["gm"]) if d["status"] else len(d["body"])) if d["copy"] else 0
        if put and cur + put > region:
            got.append(False); continue
        cur += a16(put); offs.append(rep); rep = nxt; got.append(True)
    return got, cur - region // 4, offs


def echo_request(message):
    return b"\x0a" + varint(len(message)) + message


def mutation_corpus(n, seed=3):
    """n raw request messages: well-formed EchoRequests and the mutations a client can send through an identity serializer"""
    import random
    rng = random.Random(seed)
    out = []
    for i in range(n):
        m = bytes(rng.randrange(97, 123) for _ in range([0, 1, 5, 127, 128, 300, 4096, 20000][i % 8]))
        kind = i % 9
        if kind == 0: out.append(b"")                                                       # no field at all: `message` missing
        elif kind == 1: out.append(b"\x0a" + varint(len(m) + 7) + m)                        # a length past the end
        elif kind == 2: out.append(b"\x10\x05\x1a\x02zz")                                   # only unknown fields
        elif kind == 3: out.append(b"\x10\x05" + echo_request(m) + b"\x1a\x02zz")           # unknown fields around the message
        elif kind == 4: out.append(echo_request(b"first") + echo_request(m))                # repeated: the last one wins
        elif kind == 5: out.append(b"\x0a" + bytes([0x80 | (len(m) & 0x7F)]) + varint(len(m) >> 7) + m if len(m) < 128 else b"\x0a" + varint(len(m)) + m)
        elif kind == 6: out.append(b"\x8a\x00" + varint(len(m)) + m)                        # an overlong tag
        elif kind == 7: out.append(b"\x0a" + bytes([0x80 | (len(m) & 0x7F), 0x80 | ((len(m) >> 7) & 0x7F), len(m) >> 14]) + m)   # overlong length
        else: out.append(echo_request(m))
    return out


def expected_call(raw, identity=b"", request_type=b"example.EchoRequest"):
    """what a gRPC client sees for one unary call whose message is raw: ("OK", "", reply message) or (code name, details, None)"""
    ok, (off, n) = O.parse_echo_request(raw)
    if ok:
        return "OK", "", echo_request(raw[off:off + n])
    return "INVALID_ARGUMENT", error_text(identity, reason_parse(request_type)).decode(), None


def grpcio_calls(port, requests, channels=1, compression=None, in_flight=64):
    """every raw request as one Echo call through identity serializers, round-robin over `channels` channels of their own connection;
    returns (code name, details, reply) per call"""
    import threading
    import grpc
    opts = [("grpc.max_receive_message_length", 1 << 24), ("grpc.max_send_message_length", 1 << 24), ("grpc.use_local_subchannel_pool", 1)]
    chans = [grpc.insecure_channel("127.0.0.1:%d" % port, compression=compression, options=opts) for _ in range(channels)]
    try:
        calls = [ch.unary_unary("/example.EchoService/Echo", request_serializer=lambda b: b, response_deserializer=lambda b: b) for ch in chans]
        gate = threading.BoundedSemaphore(in_flight); futs = []
        for i, b in enumerate(requests):
            gate.acquire()
            f = calls[i % channels].future(b, timeout=120)
            f.add_done_callback(lambda _f: gate.release())
            futs.append(f)
        out = []
        for f in futs:
            try:
                out.append(("OK", "", f.result()))
            except grpc.RpcError as e:
                out.append((e.code().name, e.details(), None))
        return out
    finally:
        for ch in chans:
            ch.close()


class ServeConn:
    """One server connection: the C oracle's H2Conn (ParseH2Message and the reply framing, with its HPACK encoder and windows), the
    gunzip step when the connection opted in, and the serve step."""
    def __init__(self, methods=(O.ECHO_METHOD,), identity=b"", gunzip=False):
        self.methods = list(methods); self.identity = identity or b""; self.gunzip = gunzip
        self.conn = O.H2Conn(O.make_config(self.methods))

    def consume(self, b, r=0, region=1 << 30, reply_region=1 << 30, blob_used=0):
        """blob_used: the bytes the device's parse wrote behind region / 4 of run r (G.server_blob_used).  Returns dict: err, consumed, msgs
        (H2_MSG_DT, offsets into blob, flags / reserved as b2_h2_serve_batch leaves them), ctrl, blob, replies (the answered calls' bytes in
        order), answered ([bool] per message), gz ([(flags added, msg_off, inflated bytes)] per message), out_used."""
        err, cons, msgs, ctrl, blob, _, _ = self.conn.consume(b)
        msgs = msgs.copy()
        if self.gunzip:
            gz, blob_used = G.server_step(msgs, blob, None, r, region, blob_used)
        else:
            gz = [(0, None, None)] * len(msgs)
        dec = []
        for m, (add, _, got) in zip(msgs, gz):
            m["flags"] = int(m["flags"]) | add
            f = int(m["flags"])
            g = lambda o, n: bytes(blob[int(o):int(o) + int(n)])
            msg = got if f & F_GUNZIPPED else g(m["msg_off"], m["msg_len"])
            mi = int(m["method_idx"])
            dec.append(decide(f, int(m["content_type"]), self.methods[mi] if mi >= 0 else None, content_type(g(m["headers_off"], m["headers_len"])),
                              g(m["body_off"], m["body_len"]), msg, self.identity))
        answered, out_used, _ = place(dec, region, blob_used, reply_region)
        replies = []
        for m, d, a in zip(msgs, dec, answered):
            if a:
                m["flags"] = int(m["flags"]) | F_ANSWERED; m["reserved"] = d["status"]
                replies.append(self.conn.pack_response(int(m["stream_id"]), d["body"], 200, d["ct"], True, d["status"], d["gm"]))
        return dict(err=err, consumed=cons, msgs=msgs, ctrl=ctrl, blob=blob, replies=replies, answered=answered, gz=gz, out_used=out_used,
                    decisions=dec)

    def pack_host(self, m, body=b"", status=12, message=b"unimplemented"):
        """the host's reply to a call the step left alone (by default UNIMPLEMENTED, as _h2loop's engines answer)"""
        return self.conn.pack_response(int(m["stream_id"]), body, 200, b"application/grpc", True, status, message)


class OracleServeEngine:
    """_h2loop.OracleEngine with the serve step: the control bytes, the answered calls' replies, then UNIMPLEMENTED for the rest"""
    def __init__(self, identity=b"", gunzip=False, methods=(O.ECHO_METHOD,)):
        self.identity, self.gunzip, self.methods = identity, gunzip, methods
        self.conns = {}; self.n_answered = 0; self.n_errors = 0; self.n_inflated = 0

    def open(self, cid):
        self.conns[cid] = ServeConn(self.methods, self.identity, self.gunzip)

    def feed(self, cid, buf):
        c = self.conns[cid]
        res = c.consume(buf)
        host = [c.pack_host(m) for m, a in zip(res["msgs"], res["answered"]) if not a]
        f = [int(m["flags"]) for m in res["msgs"] if int(m["flags"]) & F_ANSWERED]
        self.n_answered += len(f); self.n_inflated += sum(1 for x in f if x & F_GUNZIPPED)
        self.n_errors += sum(1 for m in res["msgs"] if int(m["flags"]) & F_ANSWERED and int(m["reserved"]))
        return res["consumed"], res["ctrl"] + b"".join(res["replies"]) + b"".join(host), res["err"], len(res["msgs"])


class DeviceServeEngine:
    """the same loop on the device: one b2_h2_serve_batch per feed, then b2_h2_pack_responses for the calls it left (UNIMPLEMENTED)"""
    def __init__(self, ctx, gunzip=False):
        import threading
        self.ctx, self.gunzip = ctx, gunzip
        self.lock = threading.Lock(); self.n_answered = 0

    def open(self, cid):
        with self.lock:
            self.ctx.h2_conn_reset(cid)
            if self.gunzip:
                self.ctx.h2_conn_set_gunzip(cid)

    def feed(self, cid, buf):
        import numpy as np
        import brpc_b200
        from brpc_b200.abi import H2_RESPONSE_DT
        with self.lock:
            data, runs = brpc_b200.make_runs([buf]); runs["socket_id"] = cid
            rs, msgs, out, replies, spans = self.ctx.h2_serve_batch(data, runs, msg_cap=1024, out_cap=8 << 20, replies_cap=8 << 20)
            co, cl, so, sl = int(rs["ctrl_off"][0]), int(rs["ctrl_len"][0]), int(spans["off"][0]), int(spans["len"][0])
            reply = bytes(out[co:co + cl]) + bytes(replies[so:so + sl])
            left = msgs[(msgs["flags"] & F_ANSWERED) == 0]
            self.n_answered += int(spans["n_answered"][0])
            if len(left):
                r = np.zeros(len(left), H2_RESPONSE_DT)
                r["conn"] = cid; r["stream_id"] = left["stream_id"]; r["status_code"] = 200; r["flags"] = 1
                r["content_type_len"] = 16; r["grpc_status"] = 12; r["grpc_message_off"] = 16; r["grpc_message_len"] = 13
                reply += b"".join(self.ctx.h2_pack_responses(np.frombuffer(b"application/grpcunimplemented\0", np.uint8), r))
            return int(rs["consumed"][0]), reply, int(rs["parse_error"][0]), len(msgs)
