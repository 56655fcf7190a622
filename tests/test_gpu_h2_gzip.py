"""GPU: gzip-compressed h2 / gRPC messages inflated on the device (b2_h2_conn_set_gunzip) against the oracle (tests/_h2gzip.py), field by
field, msg_off and the inflated bytes included — on client connections (b2_h2_client_process_batch) and server connections
(b2_h2_process_batch, then a zero-copy echo of the inflated request through B2_H2_RESP_BODY_IN_OUT):
  - gzip streams with stored, fixed and dynamic blocks, an empty message, two members, trailing garbage, zlib data under "gzip",
    bit flips, truncation at every byte of a short stream, a message inflating to 1 MiB + 1;
  - header variants: gzip / GZIP / gzip twice / deflate / identity / none, the compressed flag clear under grpc-encoding: gzip,
    content-encoding: gzip on non-gRPC messages;
  - verdicts that come first (grpc-status != 0, :status 500, a bad prefix): never inflated;
  - a region too small for every inflated message: GUNZIP_HOST;
  - connections without the opt-in in the same batches: byte-identical to a context that never enabled gunzip;
  - a compressed message over 1 MiB: GUNZIP_HOST before any sizing; NO_GRPC_ENCODING only on calls that reached that check;
then gRPC C-core in both directions: the recorded capture (tests/golden/h2_gzip_capture.json.gz) replayed — server replies split across
batches, client requests through a device echo engine against the oracle echo engine byte for byte — and live: a gzip grpcio server,
1 000 calls over 8 connections, and a gzip grpcio client, 1 000 calls with up to 128 in flight, against the device echo from out."""
import gzip
import random
import zlib

import numpy as np
import pytest

import _h2client_oracle as H
import _h2gzip as G
import _oracle as O
from _h2client_cases import OK_HDRS, frame, grpc_body, lit, new_conn, trailers
from _h2client_loop import DeviceClients, OracleClients, records

pytestmark = pytest.mark.gpu
REGION = 1 << 19
PENDING, STREAM_BYTES = 64, (256 << 10) + 4096
A16 = G.a16


def _ctx(max_conns=64, pending=PENDING, stream_bytes=STREAM_BYTES):
    import brpc_b200
    ctx = brpc_b200.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 15, max_runs=512, max_resp_bytes=96 << 20)
    ctx.h2_configure(max_conns=max_conns, max_pending=pending, stream_bytes=stream_bytes)
    return ctx


def gz(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=31):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    return c.compress(data) + c.flush()


def payloads(rng):
    text = b"".join(b"field %d = %s;\n" % (i, rng.choice([b"alpha", b"beta", b"gamma"])) for i in range(400))
    return [b"", b"x", text, bytes(rng.randrange(256) for _ in range(3000)), b"\0" * 70000]


def streams(rng):
    """(name, compressed bytes) — valid streams of every block type and the damaged ones"""
    out = []
    for i, p in enumerate(payloads(rng)):
        out += [("dyn%d" % i, gz(p)), ("stored%d" % i, gz(p, level=0)), ("fixed%d" % i, gz(p, strategy=zlib.Z_FIXED))]
    base = gz(b"hello gzip world " * 40)
    short = gz(b"tiny!")
    out += [("two_members", base + gz(b"second member")), ("trailing", base + b"garbage!"), ("zlib_wrapped", gz(b"zz" * 300, wbits=15)),
            ("raw_deflate", gz(b"raw" * 100, wbits=-15)), ("python_gzip", gzip.compress(b"mtime and name" * 50)),
            ("inflates_past_1MiB", gz(b"\0" * ((1 << 20) + 1))), ("exactly_1MiB", gz(b"\1" * (1 << 20)))]
    out += [("cut%d" % k, short[:k]) for k in range(len(short))]
    for k in range(40):
        b = bytearray(base); b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        out.append(("flip%d" % k, bytes(b)))
    return out


def data_frames(sid, body, end=True):
    if not body:
        return frame(0, 1 if end else 0, sid, b"")
    out = b""
    for at in range(0, len(body), 16384):
        last = at + 16384 >= len(body)
        out += frame(0, 1 if (last and end) else 0, sid, body[at:at + 16384])
    return out


def reply(sid, hdrs, body, trl=trailers()):
    """one server reply: HEADERS, DATA, trailers (or END_STREAM on the DATA when trl is None)"""
    return frame(1, 4, sid, hdrs) + data_frames(sid, body, end=trl is None) + (frame(1, 5, sid, trl) if trl is not None else b"")


GZ_HDRS = OK_HDRS + lit(b"grpc-encoding", b"gzip")


class GzOracle(OracleClients):
    def __init__(self, n, gunzip_conns, pending=PENDING, stream_bytes=STREAM_BYTES):
        self.c = [G.GzClientConn(pending, stream_bytes, gunzip=k in gunzip_conns) for k in range(n)]


class GzDevice(DeviceClients):
    def __init__(self, ctx, conns, gunzip_conns):
        super().__init__(ctx, conns)
        for k in gunzip_conns:
            ctx.h2_conn_set_gunzip(k)

    def parse(self, chunks, region, call_cap):
        from brpc_b200.abi import RUN_DT
        data = np.frombuffer(b"".join(chunks.values()) + b"\0", np.uint8)
        runs = np.zeros(len(chunks), RUN_DT); off = 0
        for r, (k, b) in enumerate(chunks.items()):
            runs[r]["offset"] = off; runs[r]["length"] = len(b); runs[r]["socket_id"] = k; off += len(b)
        rs, calls, out = self.ctx.h2_client_process_batch(data, runs, call_cap=call_cap * len(chunks), out_cap=region * len(chunks))
        self.last = (rs, calls, out)
        res = [(int(s["parse_error"]), int(s["consumed"]), out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()) for s in rs]
        return res, [norm(c, out, data) for c in calls]


def norm(c, out, inp):
    f = int(c["flags"])
    src = inp if f & H.F_BODY_IN_INPUT else out
    msrc = out if f & G.F_GUNZIPPED else src                     # an inflated message is in out
    g = lambda buf, off, n: bytes(buf[int(off):int(off) + int(n)])
    return dict(run_idx=int(c["run_idx"]), stream_id=int(c["stream_id"]), how=int(c["how"]), status_code=int(c["status_code"]),
                error_code=int(c["error_code"]), grpc_status=int(c["grpc_status"]), flags=f,
                headers=records(g(out, c["headers_off"], c["headers_len"])), body=g(src, c["body_off"], c["body_len"]),
                msg=g(msrc, c["msg_off"], c["msg_len"]), error=g(out, c["error_off"], c["error_len"]),
                headers_off=int(c["headers_off"]), body_off=int(c["body_off"]), msg_off=int(c["msg_off"]), error_off=int(c["error_off"]))


def same(dev, orc, what):
    (drs, dcalls), (ors, ocalls) = dev, orc
    assert drs == ors, what
    assert len(dcalls) == len(ocalls), (what, len(dcalls), len(ocalls))
    for k, (d, o) in enumerate(zip(dcalls, ocalls)):
        assert d == o, (what, k, {f: (d[f], o[f]) for f in d if d[f] != o[f]})


def client_replies(cl, k, items):
    """items: (headers, body, trailers) per call, answered in order on connection k"""
    ids = new_conn(cl, k, len(items))
    return b"".join(reply(sid, h, b, t) for sid, (h, b, t) in zip(ids, items))


def client_cases(rng):
    """one list of calls per connection"""
    conns = []
    body_cases = [(GZ_HDRS, grpc_body(s, 1), trailers()) for _, s in streams(rng)]
    for at in range(0, len(body_cases), 24):
        conns.append(body_cases[at:at + 24])
    z = gz(b"header variants " * 30)
    hv = [(OK_HDRS + lit(b"grpc-encoding", e), grpc_body(z, 1), trailers()) for e in (b"gzip", b"GZIP", b"deflate", b"identity", b"gzip ", b"")]
    hv += [(OK_HDRS + lit(b"grpc-encoding", b"gzip") + lit(b"grpc-encoding", b"gzip"), grpc_body(z, 1), trailers()),
           (OK_HDRS, grpc_body(z, 1), trailers()),                                                       # no grpc-encoding: ERESPONSE
           (OK_HDRS, grpc_body(z, 1), lit(b"grpc-status", b"0") + lit(b"grpc-encoding", b"gzip")),    # in the trailers: merged
           (GZ_HDRS, grpc_body(b"plain message, flag clear", 0), trailers()),                            # uncompressed under gzip
           (GZ_HDRS, grpc_body(z, 1), trailers(b"13", b"internal%20error")),                              # grpc-status first
           (b"\x8e" + lit(b"content-type", b"application/grpc") + lit(b"grpc-encoding", b"gzip"), grpc_body(z, 1), None),   # :status 500
           (GZ_HDRS, grpc_body(z, 1)[:-1], trailers()),                                                  # invalid prefix
           (b"\x88" + lit(b"content-type", b"application/json") + lit(b"content-encoding", b"gzip"), z, None),   # not gRPC
           (b"\x88" + lit(b"content-type", b"application/json") + lit(b"content-encoding", b"gzip"), b"", None),
           (b"\x88" + lit(b"content-type", b"application/json") + lit(b"content-encoding", b"GZIP"), z, None),
           (b"\x88" + lit(b"content-type", b"application/json"), z, None)]
    conns.append(hv)
    return conns


def test_client_connections_match_the_oracle_and_leave_others_alone():
    rng = random.Random(20261015)
    cases = client_cases(rng)
    n_gz = len(cases)
    n = 2 * n_gz                                                  # the same traffic again on connections without the opt-in
    on = set(range(n_gz))
    ctx, ref = _ctx(), _ctx()
    dev = GzDevice(ctx, range(n), on); orc = GzOracle(n, on); plain = GzDevice(ref, range(n), ())
    chunks = {k: client_replies(dev, k, cases[k % n_gz]) for k in range(n)}
    assert chunks == {k: client_replies(orc, k, cases[k % n_gz]) for k in range(n)} == {k: client_replies(plain, k, cases[k % n_gz]) for k in range(n)}
    # several batches: every connection's bytes cut in three at different places
    rest = {k: b"" for k in range(n)}; got = []
    for part in range(3):
        cut = {k: chunks[k][len(chunks[k]) * part // 3:len(chunks[k]) * (part + 1) // 3] for k in range(n)}
        now = {k: rest[k] + cut[k] for k in range(n)}
        dv, ov, pv = dev.parse(now, REGION, 64), orc.parse(now, REGION, 64), plain.parse(now, REGION, 64)
        same(dv, ov, part)
        rs_on, calls_on, out_on = dev.last; rs_off, calls_off, out_off = plain.last
        for r in range(n_gz, n):                                  # the connections without the opt-in: byte-identical
            assert rs_on[r].tobytes() == rs_off[r].tobytes()
            f, c = int(rs_on[r]["first_msg"]), int(rs_on[r]["n_msgs"])
            assert calls_on[f:f + c].tobytes() == calls_off[f:f + c].tobytes()
            used = max([r * REGION + REGION // 4] + [max(int(x["headers_off"]) + A16(int(x["headers_len"])), int(x["error_off"]) + A16(int(x["error_len"])),
                                                         0 if int(x["flags"]) & H.F_BODY_IN_INPUT else int(x["body_off"]) + A16(int(x["body_len"])))
                                                     for x in calls_on[f:f + c]])
            co, cl = int(rs_on[r]["ctrl_off"]), int(rs_on[r]["ctrl_len"])
            assert np.array_equal(out_on[co:co + cl], out_off[co:co + cl])
            assert np.array_equal(out_on[r * REGION + REGION // 4:used], out_off[r * REGION + REGION // 4:used])
        for k, (perr, cons, _) in enumerate(dv[0]):
            assert perr == H.NOT_ENOUGH_DATA
            rest[k] = now[k][cons:]
        got += dv[1]
    assert all(not r for r in rest.values())
    fl = [c["flags"] for c in got if c["run_idx"] < n_gz]
    assert sum(1 for f in fl if f & G.F_GUNZIPPED) > 40 and sum(1 for f in fl if f & G.F_GUNZIP_HOST) == 2   # past 1 MiB; 1 MiB in a 512 KiB region
    assert sum(1 for f in fl if f & G.F_NO_GRPC_ENCODING) >= 1
    assert not any(c["flags"] & (G.F_GUNZIPPED | G.F_GUNZIP_HOST | G.F_NO_GRPC_ENCODING) for c in got if c["run_idx"] >= n_gz)
    assert not any(c["flags"] & G.F_GUNZIPPED and c["error_code"] for c in got)
    # what was sent comes back inflated
    by = {c["stream_id"]: c for c in got if c["run_idx"] == 0}
    p = payloads(random.Random(20261015))
    assert by[1]["msg"] == p[0] and by[7]["msg"] == p[1] and by[13]["msg"] == p[2]


def test_region_exhaustion_leaves_the_rest_to_the_host():
    """four messages of 20 000 inflated bytes in a 64 KiB region: those whose bound no longer fits are GUNZIP_HOST, a later smaller one is
    still placed"""
    sizes = [20000, 20000, 20000, 20000, 300]
    items = [(GZ_HDRS, grpc_body(gz(bytes([65 + i]) * s), 1), trailers()) for i, s in enumerate(sizes)]
    ctx = _ctx()
    dev = GzDevice(ctx, range(2), {0, 1}); orc = GzOracle(2, {0, 1})
    chunks = {k: client_replies(dev, k, items) for k in range(2)}
    assert chunks == {k: client_replies(orc, k, items) for k in range(2)}
    dv, ov = dev.parse(chunks, 1 << 16, 8), orc.parse(chunks, 1 << 16, 8)
    same(dv, ov, "exhaustion")
    fl = [c["flags"] & (G.F_GUNZIPPED | G.F_GUNZIP_HOST) for c in dv[1][:5]]
    assert G.F_GUNZIP_HOST in fl and fl[-1] == G.F_GUNZIPPED


def test_compressed_message_over_1MiB_is_left_to_the_host():
    """a stored-block stream of 1 MiB + 64 KiB compressed (kGzMaxIn exceeded before any sizing), next to a small one placed after it; plus
    a failed call (grpc-status 13) without grpc-encoding: no NO_GRPC_ENCODING flag, brpc stops at the status"""
    import os as _os
    big = gz(_os.urandom((1 << 20) + (64 << 10)), level=0)
    items = [(GZ_HDRS, grpc_body(big, 1), trailers()), (GZ_HDRS, grpc_body(gz(b"after " * 100), 1), trailers()),
             (OK_HDRS, grpc_body(gz(b"q" * 50), 1), trailers(b"13")), (OK_HDRS, grpc_body(gz(b"q" * 50), 1), trailers())]
    sb = (2 << 20) + 4096
    ctx = _ctx(8, 8, sb)
    dev = GzDevice(ctx, range(1), {0}); orc = GzOracle(1, {0}, 8, sb)
    chunks = {0: client_replies(dev, 0, items)}
    assert chunks == {0: client_replies(orc, 0, items)}
    dv, ov = dev.parse(chunks, 3 << 20, 8), orc.parse(chunks, 3 << 20, 8)
    same(dv, ov, "over 1 MiB")
    fl = [c["flags"] & (G.F_GUNZIPPED | G.F_GUNZIP_HOST | G.F_NO_GRPC_ENCODING) for c in dv[1]]
    assert fl == [G.F_GUNZIP_HOST, G.F_GUNZIPPED, 0, G.F_NO_GRPC_ENCODING], fl


def server_request(sid, path, ct, extra, body):
    hdr = b"\x83\x86" + lit(b":path", path) + lit(b"content-type", ct) + extra
    return frame(1, 4, sid, hdr) + data_frames(sid, body)


def server_cases(rng):
    z = gz(b"request body " * 50)
    ge = lit(b"grpc-encoding", b"gzip")
    per_conn = [[(b"application/grpc", ge, grpc_body(s, 1)) for _, s in streams(rng)[i::3]] for i in range(3)]
    per_conn.append([(b"application/grpc", ge, grpc_body(z, 1)), (b"application/grpc", lit(b"grpc-encoding", b"GZIP"), grpc_body(z, 1)),
                     (b"application/grpc", ge + ge, grpc_body(z, 1)), (b"application/grpc", b"", grpc_body(z, 1)),
                     (b"application/grpc", ge, grpc_body(b"small, sent plain", 0)), (b"application/grpc", ge, grpc_body(z, 1)[:-2]),
                     (b"application/grpc", lit(b"grpc-encoding", b"deflate"), grpc_body(z, 1)),
                     (b"application/json", lit(b"content-encoding", b"gzip"), z), (b"application/json", lit(b"content-encoding", b"gzip"), b""),
                     (b"application/json", lit(b"content-encoding", b"identity"), z), (b"application/grpc", ge, grpc_body(b"", 1))])
    return per_conn


def test_server_connections_match_the_oracle_and_echo_from_out():
    import brpc_b200
    from brpc_b200.abi import H2_RESPONSE_DT
    rng = random.Random(7)
    cases = server_cases(rng)
    n_gz = len(cases); n = 2 * n_gz
    ctx, ref = _ctx(), _ctx()
    for k in range(n):
        ctx.h2_conn_reset(k); ref.h2_conn_reset(k)
    for k in range(n_gz):
        ctx.h2_conn_set_gunzip(k)
    orc = [O.H2Conn() for _ in range(n)]
    streams_ = [b"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n" + frame(4, 0, 0, b"") +
                b"".join(server_request(1 + 2 * i, b"/example.EchoService/Echo", ct, ex, body) for i, (ct, ex, body) in enumerate(cases[k % n_gz]))
                for k in range(n)]
    data, runs = brpc_b200.make_runs(streams_)
    rs, msgs, out = ctx.h2_process_batch(data, runs, out_cap=n * REGION)
    rs0, msgs0, out0 = ref.h2_process_batch(data, runs, out_cap=n * REGION)
    region = (n * REGION // n) & ~63
    n_inflated = 0; resps = []; expect = []
    for r in range(n):
        f, c = int(rs[r]["first_msg"]), int(rs[r]["n_msgs"])
        d, d0 = msgs[f:f + c], msgs0[f:f + c]
        assert rs[r].tobytes() == rs0[r].tobytes()
        e, cons, om, octrl, oblob, _, _ = orc[r].consume(streams_[r])
        assert (int(rs[r]["parse_error"]), int(rs[r]["consumed"]), c) == (e, cons, len(om))
        if r >= n_gz:                                             # without the opt-in: byte-identical
            lo, hi = r * region + region // 4, r * region + region // 4 + G.server_blob_used(d0, r, region)
            co, cl = int(rs[r]["ctrl_off"]), int(rs[r]["ctrl_len"])
            assert d.tobytes() == d0.tobytes() and np.array_equal(out[lo:hi], out0[lo:hi]) and np.array_equal(out[co:co + cl], out0[co:co + cl])
            continue
        in_input = [bool(int(m["flags"]) & H.F_BODY_IN_INPUT) for m in d0]
        res, _ = G.server_step(om, oblob, in_input, r, region, G.server_blob_used(d0, r, region))
        for m, m0, (add, off, got) in zip(d, d0, res):
            assert int(m["flags"]) == int(m0["flags"]) | add, (r, int(m["stream_id"]))
            for fld in ("headers_off", "headers_len", "body_off", "body_len", "stream_id", "method_idx"):
                assert m[fld] == m0[fld]
            if off is None:
                assert (m["msg_off"], m["msg_len"]) == (m0["msg_off"], m0["msg_len"])
                continue
            assert int(m["msg_off"]) == off and bytes(out[off:off + int(m["msg_len"])]) == got
            n_inflated += 1
            resps.append((r, int(m["stream_id"]), 200, 1 | 4, 0, 16, off, len(got), 0, 0, 0, 0))   # echo from out, no copy
            expect.append(orc[r].pack_response(int(m["stream_id"]), got, 200, b"application/grpc", True, 0, b""))
    assert n_inflated > 30
    got = ctx.h2_pack_responses(np.frombuffer(b"application/grpc\0", np.uint8), np.array(resps, dtype=H2_RESPONSE_DT))
    assert got == expect


def test_reset_clears_the_opt_in():
    ctx = _ctx()
    ctx.h2_client_conn_reset(0); ctx.h2_conn_set_gunzip(0); ctx.h2_client_conn_reset(0)
    orc = GzOracle(1, ())
    dev = DeviceClients(ctx, ())
    items = [(GZ_HDRS, grpc_body(gz(b"abc" * 100), 1), trailers())]
    chunks = {0: client_replies(dev, 0, items)}
    assert chunks == {0: client_replies(orc, 0, items)}
    dv, ov = dev.parse(chunks, REGION, 8), orc.parse(chunks, REGION, 8)
    same(dv, ov, "reset")
    assert len(dv[1]) == 1 and dv[1][0]["flags"] & H.F_COMPRESSED and not dv[1][0]["flags"] & G.F_GUNZIPPED


def test_live_gzip_grpcio_server():
    """1000 echo calls over 8 connections to a grpcio server with compression=Gzip; the device parses the replies and inflates them, only
    what the parser wrote back goes to the server.  Every reply equals its request; compressed replies actually occurred."""
    pytest.importorskip("grpc")
    import socket
    from _h2client_loop import ECHO, GRPC_EXTRA, run_socket
    srv, port = G.gzip_grpcio_server()
    ctx = _ctx(8, 128, (128 << 10) + 4096)
    n = 0; n_gz = 0
    try:
        for k in range(8):
            dev = GzDevice(ctx, [k], [k])
            with socket.create_connection(("127.0.0.1", port)) as s:
                s.settimeout(60)
                batches = [[(ECHO, b"first", GRPC_EXTRA)]]
                for b in range(5):
                    batch = []
                    for i in range(25):
                        q = k * 125 + b * 25 + i
                        size = [0, 7, 300, 4096, 20000, 70000][q % 6]
                        body = (b"echo %d " % q * (size // 6 + 1))[:size] if q % 3 else bytes((q * 7 + j * j) & 0xff for j in range(size))
                        batch.append((ECHO, body, GRPC_EXTRA))
                    batches.append(batch)
                done = run_socket(dev, s, k, batches)
            sent = [c for bt in batches for c in bt]
            assert len(done) == len(sent)
            for sid, (_, body, _) in zip(sorted(done), sent):
                c = done[sid]
                assert c["error_code"] == 0 and c["msg"] == body, (k, sid, len(body))
                assert not c["flags"] & G.F_GUNZIP_HOST
                n_gz += bool(c["flags"] & G.F_GUNZIPPED); n += 1
    finally:
        srv.stop(0)
    assert n == 1008 and n_gz > 300


def _capture():
    import gzip as _gzip
    import json
    import os
    with _gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "h2_gzip_capture.json.gz"), "rt") as f:
        return json.load(f)


def test_recorded_gzip_server_replies_split_across_batches():
    """the recorded reply stream of a gzip grpcio server (tests/golden/h2_gzip_capture.json.gz) on n connections at once, each segment
    between two sends cut at a different offset per connection and parsed in two batches: device == oracle, call for call"""
    cap = _capture()
    n = 24
    ctx = _ctx(n, cap["pending"], cap["stream_bytes"])
    dev = GzDevice(ctx, range(n), set(range(n))); orc = GzOracle(n, set(range(n)), cap["pending"], cap["stream_bytes"])
    steps = []
    for e in cap["client_rx"]:
        if "send" in e:
            steps.append(("send", [(bytes.fromhex(p), bytes.fromhex(b), tuple((bytes.fromhex(a), bytes.fromhex(v)) for a, v in ex)) for p, b, ex in e["send"]]))
        elif steps and steps[-1][0] == "recv":
            steps[-1] = ("recv", steps[-1][1] + bytes.fromhex(e["recv_hex"]))
        else:
            steps.append(("recv", bytes.fromhex(e["recv_hex"])))
    rest = {k: b"" for k in range(n)}; n_gz = 0; n_calls = 0; sent = []
    for j, st in enumerate(steps):
        if st[0] == "send":
            calls = [(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for k in range(n) for p, b, e in st[1]]
            assert [x[:2] for x in dev.pack(calls)] == [x[:2] for x in orc.pack(calls)]
            sent += [b for _, b, _ in st[1]]
            continue
        seg = st[1]
        for part in (0, 1):
            cut = {k: (k * 7919 + j * 104729) % (len(seg) + 1) for k in range(n)}
            chunks = {k: rest[k] + (seg[:cut[k]] if part == 0 else seg[cut[k]:]) for k in range(n)}
            dv, ov = dev.parse(chunks, 1 << 20, 64), orc.parse(chunks, 1 << 20, 64)
            same(dv, ov, (j, part))
            for k, (perr, cons, _) in enumerate(dv[0]):
                assert perr == H.NOT_ENOUGH_DATA
                rest[k] = chunks[k][cons:]
            n_calls += len(dv[1]); n_gz += sum(1 for c in dv[1] if c["flags"] & G.F_GUNZIPPED)
            for c in dv[1]:
                assert c["error_code"] == 0 and c["msg"] == sent[(c["stream_id"] - 1) // 2]
    assert n_calls == n * len(sent) and n_gz > n * 20


def test_recorded_gzip_client_requests_device_echo_equals_oracle():
    """the recorded request stream of a gzip grpcio client, in its recv() chunks, through the device engine (gunzip on, inflated requests
    echoed from out through B2_H2_RESP_BODY_IN_OUT) and the oracle engine: consumed bytes, parse status, requests and every byte written
    back identical"""
    cap = _capture()["server_rx"]
    ctx = _ctx(16, 192, 4096 + (256 << 10))
    ed, eo = G.DeviceGzEngine(ctx), G.OracleGzEngine()
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
    assert n == len(cap["bodies"]) and ed.n_gunzipped == eo.n_compressed > 30


def test_live_gzip_grpcio_client_against_the_device_echo():
    """a grpcio client with compression=Gzip: 1 000 calls, up to 128 in flight on one connection, against a TCP loop whose engine is the
    device with gunzip on, echoing the inflated requests from out: every call returns its request, compressed requests occurred"""
    pytest.importorskip("grpc")
    from _h2loop import H2LoopServer
    eng = G.DeviceGzEngine(_ctx(16, 192, 4096 + (256 << 10)))
    srv = H2LoopServer(eng)
    bodies = G.echo_bodies(1000, seed=9)
    try:
        got = G.grpcio_gzip_client_calls(srv.port, bodies, in_flight=128)
    finally:
        srv.close()
    assert got == bodies and not srv.errors, srv.errors
    assert srv.n_requests == 1000 and eng.n_gunzipped > 300, eng.n_gunzipped
