"""GPU: h2/gRPC client connections on the latency path (b2_h2_client_ring_*: k_h2_client_ring on the submit ring) against a twin context
that runs b2_h2_client_process_batch + b2_h2_pack_requests on the same tickets with the same caps — run statuses, calls, the bytes their
offsets point at, control bytes, request results and each request's frames, ticket by ticket, so that the connection state each ticket
leaves (HPACK tables, windows, deferred WINDOW_UPDATEs, the pending map, stream ids, GOAWAY) is shown equal by the next one:
  - the recorded grpcio conversation cut across tickets, each ticket also packing the next requests, one at a time and eight in flight
    (waited out of order); mutated server streams, 48 connections per ticket;
  - the shapes of a ticket (requests only, runs only, both) and the order inside one: SETTINGS / WINDOW_UPDATE before the requests they
    frame, GOAWAY before the stream ids it refuses, ended calls freeing their records before new requests take them;
  - gunzip connections, server connections in a client ticket; state calls between tickets, each counted as a relaunch;
  - every refused call while a ticket is outstanding, every capacity and argument refusal at submit;
  - idle retirement and relaunch, no launch over 100 steady tickets, one resident kernel per context in every direction;
  - a client ring context against a server ring context on the same GPU (1 000 echo calls over 8 connections, nothing mirrored by the
    host), and a live grpcio server behind a ring variant of DeviceClients."""
import gc
import gzip
import json
import os
import random
import socket
import time
import zlib

import numpy as np
import pytest

import _h2client_oracle as H
import _h2serve as S
import _oracle as O
from _h2client_cases import OK_HDRS, frame, grpc_body, lit, mutate, trailers
from _h2client_loop import ABORT, ABORT_TEXT, ECHO, GRPC_EXTRA, DeviceClients, grpcio_server, norm_device, run_socket

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MAX_BYTES = 1 << 20
REGION = 1 << 17
F_GUNZIPPED = 64


def _ctx(max_conns=64, pending=8, stream_bytes=69632, max_runs=512):
    import brpc_b200
    ctx = brpc_b200.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 15, max_runs=max_runs, max_resp_bytes=64 << 20)
    ctx.h2_configure(max_conns=max_conns, max_pending=pending, stream_bytes=stream_bytes)
    return ctx


def _err(fn, *a, **kw):
    from brpc_b200.abi import B2Error
    with pytest.raises(B2Error) as e:
        fn(*a, **kw)
    return e.value.code


def gz(b):
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    return c.compress(b) + c.flush()


def _call(k, body=b"q", path=ECHO, flags=1 | 8 | 16):
    return (k, flags, path, b"127.0.0.1:1", b"application/grpc", body, GRPC_EXTRA)


def ticket(chunks, calls):
    """{conn: bytes} and request calls (conn, flags, path, authority, content_type, body, extra) -> (data, runs, reqs): one input buffer,
    the runs' bytes first and the requests' fields behind them"""
    from brpc_b200.abi import H2_REQUEST_DT, RUN_DT
    head = b"".join(chunks.values())
    runs = np.zeros(len(chunks), RUN_DT); off = 0
    for r, (k, b) in enumerate(chunks.items()):
        runs[r]["offset"] = off; runs[r]["length"] = len(b); runs[r]["socket_id"] = k; off += len(b)
    blob, reqs = O.h2_request_blob(calls) if calls else (b"", np.zeros(0, H2_REQUEST_DT))
    reqs = reqs.astype(H2_REQUEST_DT)
    for f in ("path_off", "authority_off", "content_type_off", "body_off", "extra_off"):
        reqs[f] += len(head)
    return np.frombuffer(head + blob + b"\0", np.uint8), runs, reqs


def _snap(rs, calls, out, data):
    """what a ticket's parse defines: statuses, call records, each call's bytes (normalised), control bytes, inflated messages"""
    ctrl = [bytes(out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])]) for s in rs]
    inflated = [bytes(out[int(c["msg_off"]):int(c["msg_off"]) + int(c["msg_len"])]) for c in calls if int(c["flags"]) & F_GUNZIPPED]
    return rs.tobytes(), calls.tobytes(), [norm_device(c, out, data) for c in calls], ctrl, inflated


class Pair:
    """a ring context (b2_h2_client_ring_enable) and a twin that runs the same tickets through the two batch calls with the same caps"""
    def __init__(self, conns, pending=8, stream_bytes=69632, gunzip=(), servers=(), region=REGION, per_run=64, max_bytes=MAX_BYTES, max_reqs=256,
                 req_out_cap=4 << 20):
        self.n = n = len(conns)
        self.call_cap, self.out_cap, self.req_out_cap = per_run * n, region * n, req_out_cap
        self.ring, self.twin = _ctx(pending=pending, stream_bytes=stream_bytes), _ctx(pending=pending, stream_bytes=stream_bytes)
        for c in (self.ring, self.twin):
            for k in conns:
                c.h2_client_conn_reset(k)
                if k in gunzip:
                    c.h2_conn_set_gunzip(k)
            for k in servers:
                c.h2_conn_reset(k)
        self.ring.h2_client_ring_enable(max_bytes, self.call_cap, self.out_cap, max_reqs, req_out_cap)

    def twin_ticket(self, chunks, calls):
        data, runs, reqs = ticket(chunks, calls)
        parse = req = None
        if len(runs):
            rs, cl, out = self.twin.h2_client_process_batch(data, runs, call_cap=self.call_cap, out_cap=self.out_cap)
            parse = _snap(rs, cl, out, data)
        if len(reqs):
            res, frames = self.twin.h2_pack_requests(data, reqs, out_cap=self.req_out_cap)
            req = (res.tobytes(), frames)
        return data, runs, reqs, (parse, req)

    def check(self, got, data, want, what=""):
        rs, calls, out, res, frames = got
        parse, req = want
        if parse is None:
            assert len(rs) == 0 and len(calls) == 0, what
        else:
            g = _snap(rs, calls, out, data)
            assert g[0] == parse[0], (what, "statuses")
            assert g[1] == parse[1], (what, "calls")
            assert g[2] == parse[2], (what, "call bytes")
            assert g[3] == parse[3], (what, "ctrl")
            assert g[4] == parse[4], (what, "inflated")
        if req is None:
            assert len(res) == 0, what
        else:
            assert res.tobytes() == req[0], (what, "request results")
            assert frames == req[1], (what, "frames")

    def step(self, chunks, calls=(), what=""):
        """one ticket, waited at once; returns the ring's results"""
        data, runs, reqs, want = self.twin_ticket(chunks, list(calls))
        self.last = self.ring.h2_client_ring_submit(data, runs, reqs)
        got = self.ring.h2_client_ring_wait(self.last)
        self.check(got, data, want, what)
        return got

    def close(self):
        """at the end of every test: the pinned slots and device buffers go now, not whenever the collector finds them"""
        self.ring.close(); self.twin.close()

    def many(self, tickets, depth):
        """tickets: [(data, runs, reqs, want)] the twin ran in order; submitted `depth` at a time, each group waited last to first"""
        for i in range(0, len(tickets), depth):
            group = tickets[i:i + depth]
            ts = [self.ring.h2_client_ring_submit(d, r, q) for d, r, q, _ in group]
            for (d, r, q, want), t in reversed(list(zip(group, ts))):
                self.check(self.ring.h2_client_ring_wait(t), d, want, "ticket %d" % t)


def _capture():
    cap = json.load(gzip.open(os.path.join(HERE, "golden", "h2_client_rx_capture.json.gz"), "rt"))
    steps = []
    for e in cap["events"]:
        if "send" in e:
            steps.append(("send", [(bytes.fromhex(p), bytes.fromhex(b), tuple((bytes.fromhex(n), bytes.fromhex(v)) for n, v in ex))
                                   for p, b, ex in e["send"]], bytes.fromhex(e["wire_hex"])))
        elif steps and steps[-1][0] == "recv":
            steps[-1] = ("recv", steps[-1][1] + bytes.fromhex(e["recv_hex"]))
        else:
            steps.append(("recv", bytes.fromhex(e["recv_hex"])))
    return cap, steps


def _sends(st, live):
    return [(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for k in live for p, b, e in st[1]]


@pytest.mark.parametrize("depth", [1, 8])
def test_recorded_conversation_across_tickets_equals_the_batch_calls(depth):
    """The recorded server byte stream on n connections, each received segment cut in two at a different offset per connection; the
    second piece goes in the same ticket as the next send's requests.  The first ticket carries requests only."""
    from brpc_b200.abi import H2_RUN_STATUS_DT
    cap, steps = _capture()
    n = 8
    pair = Pair(range(n), cap["pending"], cap["stream_bytes"], region=1 << 19, per_run=128, max_bytes=4 << 20, max_reqs=1024)
    queued = _sends(steps[0], range(n))
    tk = pair.twin_ticket({}, queued)                                # requests only: preface, SETTINGS, WINDOW_UPDATE, the calls
    assert b"".join(tk[3][1][1][:len(steps[0][1])]) == steps[0][2]  # connection 0 sends what was recorded
    tickets = [tk]; n_reqs = len(queued)
    rest = {k: b"" for k in range(n)}
    for j in range(1, len(steps)):
        if steps[j][0] == "send":
            continue
        seg = steps[j][1]
        nxt = steps[j + 1] if j + 1 < len(steps) else None           # (received segments are merged: the next step is a send)
        cuts = {k: (k * 7919 + j * 104729) % (len(seg) + 1) for k in range(n)}
        for part in (0, 1):
            chunks = {k: rest[k] + (seg[:cuts[k]] if part == 0 else seg[cuts[k]:]) for k in range(n)}
            calls = _sends(nxt, range(n)) if part == 1 and nxt else []
            tk = pair.twin_ticket(chunks, calls)
            tickets.append(tk); n_reqs += len(calls)
            rs = np.frombuffer(tk[3][0][0], H2_RUN_STATUS_DT)
            for k in range(n):
                assert int(rs[k]["parse_error"]) == H.NOT_ENOUGH_DATA, (j, part, k)
                rest[k] = chunks[k][int(rs[k]["consumed"]):]
    assert all(not r for r in rest.values())
    parsed = [c for t in tickets if t[3][0] for c in t[3][0][2]]
    assert len(parsed) == n_reqs and sum(c["error_code"] == 0 and c["grpc_status"] == 0 for c in parsed) > n * 100
    pair.many(tickets, depth)
    pair.close()



def test_mutated_server_streams_48_connections_per_ticket():
    """The recorded conversation on 48 connections in lockstep; at one received segment each connection gets its own mutation of it
    (tests/_h2client_cases.mutate), then the conversation goes on, every ticket also packing the next send of the live connections."""
    from brpc_b200.abi import H2_RUN_STATUS_DT
    cap, steps = _capture()
    recv_at = [j for j, s in enumerate(steps) if s[0] == "recv"]
    rng = random.Random(20261017)
    n = 48; n_calls = 0; n_errors = 0
    for j in recv_at[:3]:
        end = min(j + 3, len(steps))
        pair = Pair(range(n), cap["pending"], cap["stream_bytes"], per_run=128)
        rest = {k: b"" for k in range(n)}
        got = pair.step({}, _sends(steps[0], range(n)), what=(j, 0))
        ids = sorted({int(s) for s in got[3]["stream_id"]})
        for jj in range(1, end):
            st = steps[jj]
            if st[0] == "send":                                      # (packed with the segment before it)
                continue
            live = [k for k in range(n) if rest[k] is not None]
            chunks = {k: rest[k] + (mutate(rng, st[1], ids) if jj == j else st[1]) for k in live}
            nxt = steps[jj + 1] if jj + 1 < end else None
            got = pair.step(chunks, _sends(nxt, live) if nxt else [], what=(j, jj))
            if len(got[3]):
                ids = sorted({int(s) for s in got[3]["stream_id"]})
            n_calls += len(got[1])
            for k, s in zip(live, np.array(got[0], copy=True).view(H2_RUN_STATUS_DT)):
                if int(s["parse_error"]) == H.NOT_ENOUGH_DATA:
                    rest[k] = chunks[k][int(s["consumed"]):]
                else:
                    rest[k] = None; n_errors += 1
        pair.close()
    assert n_calls > 200 and n_errors > 3


def test_ticket_shapes():
    """requests only (the preface, SETTINGS and WINDOW_UPDATE go out with the first one), runs only, both"""
    pair = Pair(range(2))
    got = pair.step({}, [_call(0), _call(0), _call(1)], what="requests only")
    res, frames = got[3], got[4]
    assert [int(r["stream_id"]) for r in res] == [1, 3, 1] and (res["status"] == H.REQ_OK).all()
    assert frames[0].startswith(b"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n") and frames[2].startswith(b"PRI * HTTP/2.0")
    assert not frames[1].startswith(b"PRI")
    got = pair.step({0: frame(4, 0, 0, b"") + frame(1, 5, 1, OK_HDRS + trailers())}, (), what="runs only")
    assert len(got[1]) == 1 and len(got[3]) == 0 and int(got[0][0]["ctrl_len"]) > 0
    got = pair.step({0: frame(1, 5, 3, OK_HDRS + trailers()), 1: frame(1, 4, 1, OK_HDRS)}, [_call(0), _call(1, b"x" * 100)], what="both")
    assert len(got[1]) == 1 and [int(r["stream_id"]) for r in got[3]] == [5, 3]
    pair.close()



def test_order_inside_a_ticket():
    """The runs of a ticket act before its requests: SETTINGS_INITIAL_WINDOW_SIZE and WINDOW_UPDATE decide ELIMIT, GOAWAY decides LOGOFF,
    calls that end free their records so that NO_ROOM does not occur."""
    pair = Pair(range(8), pending=2)
    pair.step({}, [_call(k) for k in range(6)] + [_call(6), _call(6), _call(7), _call(7)], what="open")
    small = frame(4, 0, 0, (4).to_bytes(2, "big") + (10).to_bytes(4, "big"))
    large = frame(4, 0, 0, (4).to_bytes(2, "big") + (1 << 20).to_bytes(4, "big")) + frame(8, 0, 0, (1 << 20).to_bytes(4, "big"))
    # (until the server's first SETTINGS the windows are maximised; that frame brings the connection window down to 65535)
    chunks = {0: small, 1: large, 2: frame(4, 0, 0, b""), 3: frame(7, 0, 0, (1).to_bytes(4, "big") + bytes(4)), 5: large[:15],
              6: frame(1, 5, 1, OK_HDRS + trailers()) + frame(1, 5, 3, OK_HDRS + trailers())}
    calls = [_call(0, b"x" * 100), _call(1, b"y" * 70000), _call(2, b"y" * 70000), _call(3), _call(4), _call(5, b"y" * 70000),
             _call(6), _call(6), _call(7)]
    got = pair.step(chunks, calls, what="order")
    st = [int(r["status"]) for r in got[3]]
    assert st == [H.REQ_ELIMIT, H.REQ_OK, H.REQ_ELIMIT, H.REQ_LOGOFF, H.REQ_OK, H.REQ_ELIMIT, H.REQ_OK, H.REQ_OK, H.REQ_NO_ROOM], st
    pair.step({1: frame(1, 5, 3, OK_HDRS + trailers())}, [_call(1, b"z" * 1000)], what="after")
    pair.close()



def test_gunzip_and_server_connections():
    """client connections with gunzip on (gzip-compressed replies inflated on the device), and server connections (b2_h2_conn_reset) in a
    client ticket: TRY_OTHERS, as with the batch call"""
    pair = Pair(range(4), gunzip={0, 2}, servers=(40, 41))
    pair.step({}, [_call(k) for k in range(4) for _ in range(3)], what="open")
    msgs = [S.echo_request(bytes(97 + (i * 7 + j) % 26 for j in range(300 + 900 * i))) for i in range(3)]
    ge = OK_HDRS + lit(b"grpc-encoding", b"gzip")
    chunks = {k: b"".join(frame(1, 4, 1 + 2 * i, ge) + frame(0, 0, 1 + 2 * i, grpc_body(gz(m), 1)) +
                         frame(1, 5, 1 + 2 * i, trailers()) for i, m in enumerate(msgs)) for k in range(4)}
    preface = b"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n" + frame(4, 0, 0, b"")
    chunks[40] = preface; chunks[41] = preface
    got = pair.step(chunks, [_call(k, b"again") for k in range(4)], what="gunzip")
    rs, calls = got[0], got[1]
    assert [int(s["parse_error"]) for s in rs[4:]] == [H.TRY_OTHERS] * 2
    assert int(np.count_nonzero(calls["flags"] & F_GUNZIPPED)) == 2 * len(msgs)
    for c in calls[(calls["flags"] & F_GUNZIPPED) != 0]:
        assert got[2][int(c["msg_off"]):int(c["msg_off"]) + int(c["msg_len"])].tobytes() in msgs
    assert (got[3]["status"] == H.REQ_OK).all()
    pair.close()



def test_state_calls_between_tickets(monkeypatch):
    """abandon, peer_update, set_next_stream_id, set_gunzip and conn_reset between tickets, each retiring the kernel: the next ticket
    relaunches it (counted) and still equals the batch calls"""
    gc.collect()                                                     # (no context of an earlier test is destroyed while this one counts)
    monkeypatch.setenv("B2_RING_IDLE_MS", "10000")
    n = 4
    pair = Pair(range(n))
    pair.step({}, [_call(k) for k in range(n) for _ in range(3)], what="open")
    state = [
        lambda c: c.h2_client_abandon_streams(0, [1, 3]),
        lambda c: c.h2_conn_peer_update(1, header_table_size=0, stream_window_size=1 << 20, conn_window_add=-1000),
        lambda c: c.h2_conn_set_next_stream_id(2, 101),
        lambda c: c.h2_conn_set_gunzip(3),
        lambda c: c.h2_client_conn_reset(0),
    ]
    sid = {k: 7 for k in range(n)}
    for i, f in enumerate(state):
        n0 = pair.ring.ring_launches()
        f(pair.ring); f(pair.twin)
        done = {k: frame(1, 4, sid[k] - 6, OK_HDRS) + frame(0, 0, sid[k] - 6, grpc_body(b"r%d" % i)) + frame(1, 5, sid[k] - 6, trailers())
                for k in range(1, n)}
        pair.step(done, [_call(k, b"s" * 2000) for k in range(n)], what=("state", i))
        assert pair.ring.ring_launches() == n0 + 1, i
        pair.step({k: frame(8, 0, 0, (100).to_bytes(4, "big")) for k in range(n)}, [_call(k) for k in range(n)], what=("after", i))
        assert pair.ring.ring_launches() == n0 + 1, i
        for k in range(n):
            sid[k] += 4
    pair.close()



def test_calls_refused_while_a_ticket_is_outstanding():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL, H2_REQUEST_DT, H2_RESPONSE_DT, REPLY_DT, REQUEST_DT
    pair = Pair(range(2))
    pair.step({}, [_call(0), _call(1)], what="open")
    data, runs, reqs, want = pair.twin_ticket({0: frame(1, 5, 1, OK_HDRS + trailers())}, [_call(0), _call(1)])
    ring = pair.ring
    t = ring.h2_client_ring_submit(data, runs, reqs)
    small = np.zeros(64, np.uint8)
    one_run = brpc_b200.make_runs([b"\0" * 16])
    refused = [
        lambda: ring.h2_conn_reset(0), lambda: ring.h2_conn_set_gunzip(0), lambda: ring.h2_conn_peer_update(0, stream_window_size=1000),
        lambda: ring.h2_conn_set_next_stream_id(0, 5), lambda: ring.h2_client_conn_reset(1), lambda: ring.h2_client_abandon_streams(0, [1]),
        lambda: ring.h2_process_batch(*one_run), lambda: ring.h2_serve_batch(*one_run), lambda: ring.h2_client_process_batch(*one_run),
        lambda: ring.h2_scan_batch(*one_run), lambda: ring.h2_pack_responses(small, np.zeros(1, H2_RESPONSE_DT)),
        lambda: ring.h2_pack_requests(small, np.zeros(1, H2_REQUEST_DT)), lambda: ring.hpack_reset(0),
        lambda: ring.hpack_decode_batch(small, [(0, 0, 16)]), lambda: ring.process_batch(*one_run),
        lambda: ring.crc32c_batch(small, [0], [16]), lambda: ring.snappy_compress_batch(small, [0], [16], 1024),
        lambda: ring.snappy_uncompress_batch(small, [0], [16], 1024), lambda: ring.pack_requests(small, np.zeros(1, REQUEST_DT)),
        lambda: ring.pack_responses(small, np.zeros(1, REPLY_DT)),
    ]
    for i, f in enumerate(refused):
        assert _err(f) == B2_E_INVAL, i
    pair.check(ring.h2_client_ring_wait(t), data, want, "the outstanding ticket")
    pair.step({1: frame(1, 5, 1, OK_HDRS + trailers())}, [_call(0)], what="after the refusals")
    ring.crc32c_batch(small, [0], [16])                            # between tickets every call works
    pair.step({0: frame(1, 5, 3, OK_HDRS + trailers())}, [_call(1)], what="after a call between tickets")
    pair.close()



def test_capacity_and_argument_refusals():
    from brpc_b200.abi import B2_E_CAPACITY, B2_E_INVAL
    c = _ctx()
    assert _err(c.h2_client_ring_enable, 0, 64, 1 << 20, 8, 1 << 20) == B2_E_INVAL                      # a zero cap
    assert _err(c.h2_client_ring_enable, (32 << 20) + 1, 64, 1 << 20, 8, 1 << 20) == B2_E_CAPACITY      # max_batch_bytes
    import brpc_b200
    e = brpc_b200.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 15, max_runs=512, max_resp_bytes=1 << 20)
    e.h2_configure(max_conns=8)
    assert _err(e.h2_client_ring_enable, (1 << 20) + 1, 64, 1 << 20, 8, 1 << 20) == B2_E_CAPACITY       # max_resp_bytes (b2_h2_pack_requests)
    e.close()
    assert _err(c.h2_client_ring_enable, 1 << 20, (1 << 15) + 1, 1 << 20, 8, 1 << 20) == B2_E_CAPACITY  # max_msgs
    assert _err(c.h2_client_ring_enable, 1 << 20, 64, (128 << 20) + 1, 8, 1 << 20) == B2_E_CAPACITY     # 2 * max_resp_bytes
    assert _err(c.h2_client_ring_enable, 1 << 20, 64, 1 << 20, (1 << 15) + 1, 1 << 20) == B2_E_CAPACITY # max_msgs
    assert _err(c.h2_client_ring_enable, 1 << 20, 64, 1 << 20, 8, (64 << 20) + 1) == B2_E_CAPACITY      # max_resp_bytes
    data, runs, reqs = ticket({0: b"\0" * 32}, [_call(0)])
    assert _err(c.h2_client_ring_submit, data, runs, reqs) == B2_E_INVAL                                # not enabled
    c.h2_client_ring_enable(4096, 4, 1000, 3, 1400)
    for k in range(8):
        c.h2_client_conn_reset(k)
    data, runs, reqs = ticket({k: b"\0" * 32 for k in range(5)}, [_call(0), _call(1), _call(2), _call(2)])
    assert _err(c.h2_client_ring_submit, data, runs[:0], reqs[:0]) == B2_E_INVAL                        # neither runs nor requests
    assert _err(c.h2_client_ring_submit, np.zeros(4097, np.uint8), runs[:1], reqs[:0]) == B2_E_CAPACITY # nbytes > max_bytes
    assert _err(c.h2_client_ring_submit, data, runs, reqs[:0]) == B2_E_CAPACITY                         # call_cap / n_runs == 0
    assert _err(c.h2_client_ring_submit, data, runs[:4], reqs[:0]) == B2_E_CAPACITY                     # (out_cap / 4) & ~63 < 256
    assert _err(c.h2_client_ring_submit, data, runs[:0], reqs) == B2_E_CAPACITY                         # n_reqs > max_reqs
    assert _err(c.h2_client_ring_submit, *ticket({}, [_call(0, b"x" * 1000)])) == B2_E_CAPACITY       # req_out_cap too small
    bad = runs[:2].copy(); bad["socket_id"] = 0
    assert _err(c.h2_client_ring_submit, data, bad, reqs[:0]) == B2_E_INVAL                             # one run per connection
    bad = runs[:1].copy(); bad["socket_id"] = 64
    assert _err(c.h2_client_ring_submit, data, bad, reqs[:0]) == B2_E_INVAL                             # connection out of range
    bad = runs[:1].copy(); bad["length"] = len(data) + 1
    assert _err(c.h2_client_ring_submit, data, bad, reqs[:0]) == B2_E_INVAL                             # run outside the buffer
    q = reqs[:1].copy(); q["conn"] = 64
    assert _err(c.h2_client_ring_submit, data, runs[:1], q) == B2_E_INVAL                               # request connection out of range
    q = reqs[:1].copy(); q["body_len"] = len(data)
    assert _err(c.h2_client_ring_submit, data, runs[:1], q) == B2_E_INVAL                               # body outside the buffer
    q = reqs[:1].copy(); q["extra_len"] -= 1
    assert _err(c.h2_client_ring_submit, data, runs[:1], q) == B2_E_INVAL                               # truncated extra header record
    long_path = ticket({}, [(0, 1 | 8 | 16, b"/" * 1100, b"h:1", b"application/grpc", b"q", ())])
    assert _err(c.h2_client_ring_submit, *long_path) == B2_E_INVAL                                      # header block too long
    q = np.concatenate([reqs[:1], reqs[1:2], reqs[:1]])
    assert _err(c.h2_client_ring_submit, data, runs[:0], q) == B2_E_INVAL                               # one connection's requests apart
    # after the refusals the ring takes tickets, and a full ring refuses the ninth
    ts = [c.h2_client_ring_submit(data, runs[k:k + 1], reqs[:0]) for k in range(5)] + [c.h2_client_ring_submit(data, runs[:0], reqs[k:k + 1]) for k in range(3)]
    assert _err(c.h2_client_ring_submit, data, runs[:1], reqs[:0]) == B2_E_CAPACITY                     # eight outstanding
    for t in ts:
        c.h2_client_ring_wait(t)
    assert _err(c.h2_client_ring_wait, ts[0]) == B2_E_INVAL                                             # already collected
    c.close()


def _steady(pair, sid, steps):
    """a steady client loop: each ticket reads the replies to the previous requests and sends the next ones"""
    for _ in range(steps):
        chunks = {k: frame(1, 4, sid[k], OK_HDRS) + frame(0, 0, sid[k], grpc_body(b"ok")) + frame(1, 5, sid[k], trailers()) for k in range(pair.n)}
        got = pair.step(chunks, [_call(k, b"steady" * 20) for k in range(pair.n)])
        assert len(got[1]) == pair.n and (got[1]["error_code"] == 0).all()
        for k in range(pair.n):
            sid[k] += 2


def test_idle_retirement_relaunch_and_no_launch_over_100_steady_tickets(monkeypatch):
    gc.collect()                                                     # (no context of an earlier test is destroyed while this one counts)
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    pair = Pair(range(4))
    pair.step({}, [_call(k) for k in range(4)])
    sid = [1] * 4
    n0 = pair.ring.ring_launches()
    _steady(pair, sid, 100)
    assert pair.ring.ring_launches() == n0
    pair.ring.ring_stop()
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    _steady(pair, sid, 1)                                           # relaunched by the submission, now with a 5 ms idle time
    n1 = pair.ring.ring_launches()
    assert n1 == n0 + 1
    time.sleep(0.2)                                                  # it retires and comes back with the next submission
    _steady(pair, sid, 2)
    assert pair.ring.ring_launches() > n1
    ph = pair.ring.ring_phase_ns(pair.last)
    assert 0 < ph[0] <= ph[1] <= ph[2] <= ph[3]
    pair.close()



def test_one_resident_kernel_per_context():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL
    caps = (1 << 20, 64, 1 << 20, 16, 1 << 20)
    a = _ctx(); a.ring_start()
    assert _err(a.h2_client_ring_enable, *caps) == B2_E_INVAL                                           # after k_ring
    a.ring_stop()
    b = _ctx(); b.h2_ring_enable(1 << 20, 64, 1 << 20, 1 << 20)
    assert _err(b.h2_client_ring_enable, *caps) == B2_E_INVAL                                           # after k_h2_ring
    c = _ctx(); c.stream_configure(64, 1 << 16); c.stream_ring_enable(1 << 16)
    assert _err(c.h2_client_ring_enable, *caps) == B2_E_INVAL                                           # with the stream pass on k_ring
    d = _ctx(); d.h2_client_ring_enable(*caps)
    assert _err(d.h2_client_ring_enable, *caps) == B2_E_INVAL                                           # twice
    assert _err(d.h2_ring_enable, 1 << 20, 64, 1 << 20, 1 << 20) == B2_E_INVAL
    assert _err(d.h2_configure, 8) == B2_E_INVAL                                                        # enable comes after b2_h2_configure
    d.stream_configure(64, 1 << 16)
    assert _err(d.stream_ring_enable, 1 << 16) == B2_E_INVAL
    assert _err(d.h2_client_ring_wait, 1) == B2_E_INVAL                                                 # no such ticket
    data, runs = brpc_b200.make_runs([b"\0" * 16])
    assert _err(d.h2_ring_submit, data, runs) == B2_E_INVAL
    e = _ctx(); e.h2_client_ring_enable(*caps)
    assert _err(e.ring_submit, data, runs) == B2_E_INVAL
    e.h2_client_conn_reset(0)
    data, runs, reqs = ticket({}, [_call(0)])
    t = e.h2_client_ring_submit(data, runs, reqs)
    assert _err(e.ring_wait, t) == B2_E_INVAL and _err(e.h2_ring_wait, t) == B2_E_INVAL
    assert int(e.h2_client_ring_wait(t)[3]["status"][0]) == H.REQ_OK
    for x in (a, b, c, d, e):
        x.close()


def test_device_round_trip_client_ring_against_server_ring():
    """1 000 echo calls over 8 connections between a client ring context and a server ring context (k_h2_ring with device echo) on the
    same GPU: each side's wire bytes are only what its kernel wrote (control bytes, request frames, replies)."""
    from test_gpu_h2_serve import IDENTITY, METHODS, _ctx as server_ctx
    n, per_round, rounds = 8, 25, 5
    cli = _ctx(pending=64, stream_bytes=16384)
    srv = server_ctx(METHODS, IDENTITY)
    for k in range(n):
        cli.h2_client_conn_reset(k); srv.h2_conn_reset(k)
    cli.h2_client_ring_enable(MAX_BYTES, 64 * n, REGION * n, per_round * n, 4 << 20)
    srv.h2_ring_enable(MAX_BYTES, 64 * n, REGION * n, REGION * n)
    sent = {}; done = {}; to_srv = {k: b"" for k in range(n)}; to_cli = {k: b"" for k in range(n)}
    rng = random.Random(11)
    for rnd in range(rounds + 40):
        calls = []
        if rnd < rounds:
            for k in range(n):
                for _ in range(per_round):
                    calls.append(_call(k, S.echo_request(bytes(97 + rng.randrange(26) for _ in range(rng.randrange(1, 900))))))
        if not calls and not any(to_cli.values()):
            break
        chunks = {k: b for k, b in to_cli.items() if b}
        data, runs, reqs = ticket(chunks, calls)
        rs, cl, out, res, frames = cli.h2_client_ring_wait(cli.h2_client_ring_submit(data, runs, reqs))
        for r, s in zip(runs, rs):
            k = int(r["socket_id"])
            to_cli[k] = to_cli[k][int(s["consumed"]):]
            to_srv[k] += out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()
        for c in cl:
            done[(int(runs[int(c["run_idx"])]["socket_id"]), int(c["stream_id"]))] = norm_device(c, out, data)
        for q, r, f in zip(calls, res, frames):
            assert int(r["status"]) == H.REQ_OK, (rnd, int(r["status"]))
            sent[(q[0], int(r["stream_id"]))] = q[5]
            to_srv[q[0]] += f
        chunks = {k: b for k, b in to_srv.items() if b}
        if not chunks:
            continue
        data, runs = ticket(chunks, [])[:2]
        srs, msgs, sout, replies, spans = srv.h2_ring_wait(srv.h2_ring_submit(data, runs))
        assert (msgs["flags"] & S.F_ANSWERED).all()
        for r, s, sp in zip(runs, srs, spans):
            k = int(r["socket_id"])
            to_srv[k] = to_srv[k][int(s["consumed"]):]
            to_cli[k] += sout[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes() + \
                replies[int(sp["off"]):int(sp["off"]) + int(sp["len"])].tobytes()
    assert len(sent) == n * per_round * rounds == 1000
    assert sorted(done) == sorted(sent)
    for key, body in sent.items():
        c = done[key]
        assert c["how"] == H.ENDED and c["error_code"] == 0 and c["msg"] == body, key
    cli.close(); srv.close()


class RingClients(DeviceClients):
    """DeviceClients on the ring: pack is a ticket of requests, parse a ticket of runs.  A ring's caps are fixed when it is enabled, so
    the client is enabled with the caps run_socket asks for (one connection per ticket) and parse checks that it is asked for those."""
    def __init__(self, ctx, conns, region, call_cap):
        super().__init__(ctx, conns)
        self.region, self.call_cap = region, call_cap
        ctx.h2_client_ring_enable(1 << 20, call_cap, region, 128, 2 << 20)

    def pack(self, calls):
        data, runs, reqs = ticket({}, calls)
        _, _, _, res, frames = self.ctx.h2_client_ring_wait(self.ctx.h2_client_ring_submit(data, runs, reqs))
        return [(int(r["status"]), int(r["stream_id"]), f) for r, f in zip(res, frames)]

    def parse(self, chunks, region, call_cap):
        assert (len(chunks), region, call_cap) == (1, self.region, self.call_cap)
        data, runs, reqs = ticket(chunks, [])
        rs, calls, out, _, _ = self.ctx.h2_client_ring_wait(self.ctx.h2_client_ring_submit(data, runs, reqs))
        res = [(int(s["parse_error"]), int(s["consumed"]), out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()) for s in rs]
        return res, [norm_device(c, out, data) for c in calls]


def test_live_round_trip_with_a_grpcio_server():
    """1000 calls over 8 connections through run_socket (after one opening call per connection): requests packed and the server's frames
    parsed on the ring, and only what the device wrote back sent to the server"""
    pytest.importorskip("grpc")
    region, call_cap = 1 << 22, 512
    srv, port = grpcio_server()
    ctx = _ctx(8, 128, (128 << 10) + 4096)
    dev = RingClients(ctx, range(8), region, call_cap)
    n = 0
    try:
        for k in range(8):
            with socket.create_connection(("127.0.0.1", port)) as s:
                s.settimeout(60)
                first = [(ECHO, b"first", GRPC_EXTRA)]          # the server's SETTINGS come back before large bodies go out
                batches = []
                for b in range(5):
                    batch = []
                    for i in range(25):
                        q = k * 125 + b * 25 + i
                        size = [0, 7, 300, 4096, 20000, 70000][q % 6] if q % 5 else 100
                        path = ECHO if q % 17 else (ABORT if q % 2 else b"/example.Nope/Missing")
                        batch.append((path, bytes((q + j) & 0xff for j in range(size)), GRPC_EXTRA))
                    batches.append(batch)
                done = run_socket(dev, s, k, [first] + batches, region=region, call_cap=call_cap)
                sids = sorted(done)
                assert len(sids) == 1 + sum(len(b) for b in batches)
                c = done[sids[0]]
                assert (c["how"], c["error_code"], c["msg"]) == (H.ENDED, 0, b"first")
                for sid, (path, body, _) in zip(sids[1:], [c for b in batches for c in b]):
                    c = done[sid]
                    assert c["how"] == H.ENDED and c["status_code"] == 200
                    if path == ECHO:
                        assert c["error_code"] == 0 and c["msg"] == body, (k, sid, len(body))
                    elif path == ABORT:
                        assert (c["grpc_status"], c["error_code"], c["error"]) == (9, 2001, ABORT_TEXT.encode())
                    else:
                        assert (c["grpc_status"], c["error_code"]) == (12, 1002)
                    n += 1
    finally:
        srv.stop(0)
    assert n == 1000
    assert ctx.ring_launches() >= 1
    ctx.close()
