"""GPU: b2_h2_serve_batch against the serve oracle (tests/_h2serve.py) byte for byte — run statuses, messages with their flags and
grpc-status, control bytes, spans and every reply — and against a twin context that runs b2_h2_process_batch + b2_h2_pack_responses on
the same records, so that the HPACK tables, windows and deferred WINDOW_UPDATEs carried into later batches are shown equal too:
  - synthetic calls with body mutations (empty body, bad prefix, compressed without grpc-encoding, gzip, deflate, EchoRequests that do
    not parse, unknown fields, repeated and overlong fields), mixed with a host method, a gzip-replying echo method, unknown paths, JSON
    calls and an overlong content-type, on connections with and without gunzip, cut across three batches;
  - the longest error text (a 63-byte identity and a 95-byte request type: over 512 bytes of grpc-message);
  - a full reply region: the run's later calls are left, then answered by b2_h2_pack_responses, and the next batch still agrees;
  - well-formed traffic: a twin running the messenger's records (echo of the raw message, the request's content-type) gives the same bytes;
  - the recorded gzip client capture (tests/golden/h2_gzip_capture.json.gz) through the device and oracle engines;
  - a live grpcio client: 1 000 calls over 8 connections, a third of them malformed."""
import random
import zlib

import numpy as np
import pytest

import _h2serve as S
import _h2traffic as T
import _oracle as O
from _h2gzip import server_blob_used

pytestmark = pytest.mark.gpu
IDENTITY = b"10.0.0.1:8000"
REGION, RREGION = 1 << 18, 1 << 18
METHODS = (O.ECHO_METHOD, dict(O.ECHO_METHOD, method_name=b"Host", handler=0), dict(O.ECHO_METHOD, method_name=b"Gz", response_compress_type=2))


def _ctx(methods=METHODS, identity=IDENTITY, max_conns=32, pending=64, stream_bytes=(128 << 10) + 4096):
    import brpc_b200
    ctx = brpc_b200.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 15, max_runs=512, max_resp_bytes=64 << 20, methods=methods,
                            server_identity=identity)
    ctx.h2_configure(max_conns=max_conns, max_pending=pending, stream_bytes=stream_bytes)
    return ctx


def gz(b):
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    return c.compress(b) + c.flush()


def call(enc, sid, body, path=b"/example.EchoService/Echo", ct=b"application/grpc", extra=(), chunk=16000):
    """HEADERS + DATA frames of one call with a raw body (None: END_STREAM on the HEADERS, no body)"""
    block = b"".join([enc.field(b":method", b"POST"), enc.field(b":scheme", b"http"), enc.field(b":path", path),
                      enc.field(b":authority", b"127.0.0.1:8010"), enc.field(b"content-type", ct), enc.field(b"te", b"trailers")] +
                     [enc.field(n, v) for n, v in extra])
    if body is None:
        return T.frame(1, 0x5, sid, block)
    out = T.frame(1, 0x4, sid, block)
    pieces = [body[i:i + chunk] for i in range(0, len(body), chunk)] or [b""]
    for j, p in enumerate(pieces):
        out += T.frame(0, 1 if j == len(pieces) - 1 else 0, sid, p)
    return out


def prefix(pb, compressed=0, delta=0):
    return bytes([compressed]) + (len(pb) + delta).to_bytes(4, "big") + pb


def mixed_calls(rng, k):
    """(body, kwargs) per call of connection k"""
    ge = ((b"grpc-encoding", b"gzip"),)
    corpus = S.mutation_corpus(27, seed=k)
    out = [(prefix(raw), {}) for raw in corpus]
    msg = S.echo_request(b"m%d " % k * 200)
    out += [(None, {}), (prefix(msg, delta=1), {}), (prefix(msg)[:4], {}),
            (prefix(gz(msg), 1), {"extra": ge}), (prefix(gz(msg), 1), {}), (prefix(gz(msg), 1), {"extra": ((b"grpc-encoding", b"deflate"),)}),
            (prefix(gz(b"\x10\x01")), {"extra": ge}), (prefix(gz(b"\x10\x01"), 1), {"extra": ge}),
            (prefix(msg), {"path": b"/example.EchoService/Host"}), (prefix(msg), {"path": b"/example.EchoService/Gz"}),
            (prefix(msg), {"path": b"/other.Service/Echo"}), (prefix(msg), {"ct": b"application/grpc+json"}),
            (prefix(msg), {"ct": b"application/grpc+proto;" + b"x" * 300}), (prefix(msg), {"ct": b"application/grpc+proto"}),
            (prefix(S.echo_request(bytes(rng.randrange(256) for _ in range(40000)))), {}), (prefix(msg), {"chunk": 100})]
    rng.shuffle(out)
    return out


WINDOW = T.frame(8, 0, 0, (1 << 30).to_bytes(4, "big"))             # the client's connection window: room for every reply


def conn_stream(rng, k, calls):
    enc = T.HpackEncoder(rng)
    return T.PREFACE + T.settings() + WINDOW + b"".join(call(enc, 1 + 2 * i, b, **kw) for i, (b, kw) in enumerate(calls))


def host_records(items):
    """b2_h2_response records + their bytes for (conn, stream_id, ct, body, grpc_status, grpc_message)"""
    from brpc_b200.abi import H2_RESPONSE_DT
    blob = b""; r = np.zeros(len(items), H2_RESPONSE_DT)
    for i, (conn, sid, ct, body, st, gm) in enumerate(items):
        r[i] = (conn, sid, 200, 1, len(blob), len(ct), len(blob) + len(ct), len(body), st, len(blob) + len(ct) + len(body), len(gm), 0)
        blob += ct + body + gm
    return np.frombuffer(blob + b"\0" * 16, np.uint8), r


class Trio:
    """the device (b2_h2_serve_batch), a twin context (b2_h2_process_batch + b2_h2_pack_responses of the same records) and the oracle"""
    def __init__(self, n, gunzip=(), methods=METHODS, identity=IDENTITY):
        self.dev, self.twin = _ctx(methods, identity), _ctx(methods, identity)
        self.orc = [S.ServeConn(methods, identity, gunzip=k in gunzip) for k in range(n)]
        for k in range(n):
            for c in (self.dev, self.twin):
                c.h2_conn_reset(k)
                if k in gunzip:
                    c.h2_conn_set_gunzip(k)

    def batch(self, chunks, region=REGION, rregion=RREGION):
        """one batch; asserts everything equal; returns (consumed per run, answered count, left count)"""
        import brpc_b200
        n = len(chunks)
        data, runs = brpc_b200.make_runs(chunks)
        runs["socket_id"] = np.arange(n)
        rs, msgs, out, replies, spans = self.dev.h2_serve_batch(data, runs, msg_cap=n * 128, out_cap=n * region, replies_cap=n * rregion)
        rs0, msgs0, out0 = self.twin.h2_process_batch(data, runs, msg_cap=n * 128, out_cap=n * region)
        assert rs.tobytes() == rs0.tobytes()
        assert len(msgs) == len(msgs0)
        for fld in msgs.dtype.names:                              # everything but the answered flag and the grpc-status
            if fld not in ("flags", "reserved"):
                assert np.array_equal(msgs[fld], msgs0[fld]), fld
        cons, twin_items, left, n_ans = [], [], [], 0
        for r in range(n):
            f, c = int(rs[r]["first_msg"]), int(rs[r]["n_msgs"])
            d, d0 = msgs[f:f + c], msgs0[f:f + c]
            res = self.orc[r].consume(chunks[r], r, region, rregion, server_blob_used(d0, r, region))
            assert (res["err"], res["consumed"], len(res["msgs"])) == (int(rs[r]["parse_error"]), int(rs[r]["consumed"]), c)
            co, cl = int(rs[r]["ctrl_off"]), int(rs[r]["ctrl_len"])
            assert bytes(out[co:co + cl]) == bytes(out0[co:co + cl]) == res["ctrl"], r
            for m, m0, a, dec in zip(d, d0, res["answered"], res["decisions"]):
                assert int(m["flags"]) == int(m0["flags"]) | (S.F_ANSWERED if a else 0), (r, int(m["stream_id"]))
                assert int(m["reserved"]) == (dec["status"] if a else 0)
                if a:
                    ct = S.content_type(bytes(out0[int(m0["headers_off"]):int(m0["headers_off"]) + int(m0["headers_len"])]))
                    twin_items.append((r, int(m["stream_id"]), ct, dec["body"], dec["status"], dec["gm"]))
                else:
                    left.append((r, m, m0))
            so, sl = int(spans[r]["off"]), int(spans[r]["len"])
            assert (so, int(spans[r]["n_answered"])) == (r * rregion, len(res["replies"])), r
            assert bytes(replies[so:so + sl]) == b"".join(res["replies"]), r
            n_ans += len(res["replies"]); cons.append(int(rs[r]["consumed"]))
        if twin_items and all(len(x[5]) <= 512 for x in twin_items):   # (the host call takes at most 512 bytes of grpc-message)
            tb, tr = host_records(twin_items)
            assert b"".join(self.twin.h2_pack_responses(tb, tr)) == b"".join(bytes(replies[int(s["off"]):int(s["off"]) + int(s["len"])]) for s in spans)
        if left:                                                  # the host answers the rest on all three, UNIMPLEMENTED
            hb, hr = host_records([(r, int(m["stream_id"]), b"application/grpc", b"", 12, b"unimplemented") for r, m, _ in left])
            got_dev, got_twin = self.dev.h2_pack_responses(hb, hr), self.twin.h2_pack_responses(hb, hr)
            got_orc = [self.orc[r].pack_host(m0) for r, _, m0 in left]
            assert got_dev == got_twin == got_orc
        return cons, n_ans, len(left)


def _cut_batches(trio, streams, parts=3):
    n = len(streams); rest = [b""] * n; n_ans = n_left = 0
    for part in range(parts):
        now = [rest[k] + streams[k][len(streams[k]) * part // parts:len(streams[k]) * (part + 1) // parts] for k in range(n)]
        cons, a, l = trio.batch(now)
        rest = [now[k][cons[k]:] for k in range(n)]; n_ans += a; n_left += l
    assert not any(rest)
    return n_ans, n_left


def test_mixed_calls_across_batches_match_the_oracle_and_the_twin():
    rng = random.Random(20261016)
    n = 16
    trio = Trio(n, gunzip=set(range(0, n, 2)))
    streams = [conn_stream(rng, k, mixed_calls(rng, k)) for k in range(n)]
    n_ans, n_left = _cut_batches(trio, streams)
    assert n_ans > 30 * n and n_left > 6 * n


def test_longest_error_text():
    """an identity and a request type of 63 and 95 digits (each escaped to three bytes): a grpc-message past the 512 bytes
    b2_h2_pack_responses takes from the host, within what k_h2_pack's buffers hold (702, every byte escaped)"""
    rt = b"0" * 95
    methods = (dict(O.ECHO_METHOD, request_type_name=rt),)
    trio = Trio(2, methods=methods, identity=b"9" * 63)
    enc = T.HpackEncoder(random.Random(1))
    enc2 = T.HpackEncoder(random.Random(1))
    streams = [T.PREFACE + T.settings() + call(enc, 1, None) + call(enc, 3, prefix(b"\x10")),
               T.PREFACE + T.settings() + call(enc2, 1, None) + call(enc2, 3, None)]
    _, n_ans, _ = trio.batch(streams)
    assert n_ans == 4
    text = S.percent_encode(S.error_text(b"9" * 63, S.reason_empty(rt)))
    assert 512 < len(text) <= 702


def test_full_reply_region_leaves_the_rest_to_the_host():
    rng = random.Random(5)
    n = 4
    trio = Trio(n)
    msgs = [S.echo_request(bytes(rng.randrange(97, 123) for _ in range(3000))) for _ in range(12)]
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    first = [T.PREFACE + T.settings() + WINDOW + b"".join(call(enc[k], 1 + 2 * i, prefix(m)) for i, m in enumerate(msgs)) for k in range(n)]
    _, n_ans, n_left = trio.batch(first, rregion=4 * 4096)       # three or so replies fit each run's region
    assert 0 < n_ans < n * 6 and n_left == n * 12 - n_ans
    nxt = [b"".join(call(enc[k], 25 + 2 * i, prefix(m)) for i, m in enumerate(msgs)) for k in range(n)]
    _, n_ans2, n_left2 = trio.batch(nxt)                           # the state the host's replies left is the device's
    assert n_ans2 == n * 12 and n_left2 == 0


def test_well_formed_traffic_equals_the_messenger_records():
    """grpc_h2-like traffic (4 KB messages, HPACK table hits, K calls per connection): the replies of b2_h2_serve_batch equal a twin's
    b2_h2_pack_responses of the records GpuH2Messenger builds (raw message echoed from the device, the request's content-type), batch
    after batch"""
    import brpc_b200
    from brpc_b200.abi import H2_RESPONSE_DT
    rng = random.Random(11)
    n, K = 32, 8
    dev, twin = _ctx(), _ctx()
    message = bytes(rng.choice(b"abcdefghij") for _ in range(4096))
    encs = [T.HpackEncoder(rng) for _ in range(n)]
    for e in encs:
        e.fixed_mode = "auto"
    for k in range(n):
        dev.h2_conn_reset(k); twin.h2_conn_reset(k)
    sid = [1] * n
    for step in range(3):
        chunks = []
        for k in range(n):
            b = (T.PREFACE + T.settings() if step == 0 else T.frame(8, 0, 0, (K * 5000).to_bytes(4, "big")))
            for _ in range(K):
                b += b"".join(T.request_frames(rng, encs[k], sid[k], message=message, chunk=rng.choice([16384, 1000]))); sid[k] += 2
            chunks.append(b)
        data, runs = brpc_b200.make_runs(chunks); runs["socket_id"] = np.arange(n)
        rs, msgs, out, replies, spans = dev.h2_serve_batch(data, runs, msg_cap=n * 64, out_cap=n * REGION, replies_cap=n * RREGION)
        rs0, msgs0, out0 = twin.h2_process_batch(data, runs, msg_cap=n * 64, out_cap=n * REGION)
        assert len(msgs) == n * K and np.all(msgs["flags"] & S.F_ANSWERED) and not np.any(msgs["reserved"])
        r = np.zeros(len(msgs0), H2_RESPONSE_DT)
        r["conn"] = runs["socket_id"][msgs0["run_idx"]]; r["stream_id"] = msgs0["stream_id"]; r["status_code"] = 200
        r["flags"] = 1 | 8 | np.where(msgs0["flags"] & 16, 2, 4)
        for i, m in enumerate(msgs0):                              # FindHeader: the last content-type record
            h = bytes(out0[int(m["headers_off"]):int(m["headers_off"]) + int(m["headers_len"])])
            p = 0
            while p < len(h):
                nl, vl = h[p] | (h[p + 1] << 8), h[p + 2] | (h[p + 3] << 8)
                if h[p + 4:p + 4 + nl] == b"content-type":
                    r[i]["content_type_off"] = int(m["headers_off"]) + p + 4 + nl; r[i]["content_type_len"] = vl
                p += 4 + nl + vl
        r["body_off"] = msgs0["msg_off"]; r["body_len"] = msgs0["msg_len"]
        want = twin.h2_pack_responses(None, r)
        got = [bytes(replies[int(s["off"]):int(s["off"]) + int(s["len"])]) for s in spans]
        per_run = [b"".join(want[int(rs0[q]["first_msg"]):int(rs0[q]["first_msg"]) + int(rs0[q]["n_msgs"])]) for q in range(n)]
        assert got == per_run, step
        for q in range(n):
            co, cl = int(rs[q]["ctrl_off"]), int(rs[q]["ctrl_len"])
            assert bytes(out[co:co + cl]) == bytes(out0[co:co + cl])


def test_recorded_gzip_client_capture_equals_the_oracle_engine():
    import gzip
    import json
    import os
    with gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "h2_gzip_capture.json.gz"), "rt") as f:
        cap = json.load(f)["server_rx"]
    ed = S.DeviceServeEngine(_ctx((O.ECHO_METHOD,), b"", 16, 192, 4096 + (256 << 10)), gunzip=True); eo = S.OracleServeEngine(gunzip=True)
    n = 0
    for cid, chunks in cap["chunks"].items():
        cid = int(cid); ed.open(cid); eo.open(cid)
        pd = po = b""
        for i, ch in enumerate(chunks):
            ch = bytes.fromhex(ch); pd += ch; po += ch
            cd, od, errd, nd = ed.feed(cid, pd)
            co, oo, erro, no = eo.feed(cid, po)
            assert (cd, errd, nd) == (co, erro, no) and od == oo, (cid, i)
            pd = pd[cd:]; po = po[co:]; n += nd
    assert n == len(cap["bodies"]) and ed.n_answered == eo.n_answered and eo.n_inflated > 30


def test_live_grpcio_client_1000_calls_over_8_connections():
    pytest.importorskip("grpc")
    from _h2loop import H2LoopServer
    eng = S.DeviceServeEngine(_ctx((O.ECHO_METHOD,), IDENTITY, 16, 128))
    srv = H2LoopServer(eng)
    reqs = S.mutation_corpus(1000, seed=8)
    try:
        got = S.grpcio_calls(srv.port, reqs, channels=8)
    finally:
        srv.close()
    assert not srv.errors, srv.errors
    assert got == [S.expected_call(r, IDENTITY) for r in reqs]
    assert eng.n_answered == 1000 and sum(1 for g in got if g[0] != "OK") > 200
