"""GPU: the receiving half of h2 client connections on the device (b2_h2_client_conn_reset, b2_h2_pack_requests on such connections,
b2_h2_client_process_batch, b2_h2_client_abandon_streams) against the oracle (tests/_h2client_oracle.py, pinned by a grpcio server in
tests/test_oracle_h2_client_rx_grpcio.py), call for call: every b2_h2_call field, the bytes its offsets point at, the ctrl bytes and the
run status — on a recorded grpcio conversation split at many offsets across batches, on hand-built frames, at the pool's limits and next
to server connections in the same batch; then a live round trip with a grpcio server where nothing is mirrored by the host."""
import gzip
import json
import os
import socket

import numpy as np
import pytest

import _h2client_oracle as H
from _h2client_cases import HAND_CASES, STREAM_BYTES
from _h2client_loop import ABORT, ABORT_TEXT, ECHO, GRPC_EXTRA, DeviceClients, OracleClients, grpcio_server, run_socket

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
REGION = 1 << 19


def _ctx(max_conns, pending, stream_bytes):
    import brpc_b200
    ctx = brpc_b200.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 15, max_runs=512, max_resp_bytes=96 << 20)
    ctx.h2_configure(max_conns=max_conns, max_pending=pending, stream_bytes=stream_bytes)
    return ctx


def same(dev, orc, what):
    (drs, dcalls), (ors, ocalls) = dev, orc
    assert drs == ors, (what, [(a[:2], b[:2]) for a, b in zip(drs, ors) if a != b][:3])
    assert len(dcalls) == len(ocalls), (what, len(dcalls), len(ocalls))
    for k, (d, o) in enumerate(zip(dcalls, ocalls)):
        assert d == o, (what, k, {f: (d[f], o[f]) for f in d if d[f] != o[f]})


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


def test_recorded_grpcio_conversation_split_everywhere():
    """The recorded server byte stream on n connections at once, each segment between two sends cut at a different offset per connection
    (every offset of the first segments, spread over the long ones), the pieces parsed in consecutive batches."""
    cap, steps = _capture()
    n = 160
    ctx = _ctx(n, cap["pending"], cap["stream_bytes"])
    dev = DeviceClients(ctx, range(n)); orc = OracleClients(n, cap["pending"], cap["stream_bytes"])
    rest = {k: b"" for k in range(n)}
    n_calls = 0; ok = 0; n_sent = 0
    for j, st in enumerate(steps):
        if st[0] == "send":
            calls = [(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for k in range(n) for p, b, e in st[1]]
            d, o = dev.pack(calls), orc.pack(calls)
            assert d == o and b"".join(x[2] for x in d[:len(st[1])]) == st[2], j     # connection 0 sends what was recorded
            n_sent += len(st[1])
            continue
        seg = st[1]
        cuts = {k: (k if j < 4 else (k * 7919 + j * 104729)) % (len(seg) + 1) for k in range(n)}
        for part in (0, 1):
            chunks = {k: rest[k] + (seg[:cuts[k]] if part == 0 else seg[cuts[k]:]) for k in range(n)}
            dv, ov = dev.parse(chunks, REGION, 128), orc.parse(chunks, REGION, 128)
            same(dv, ov, (j, part))
            for k, (perr, cons, _) in enumerate(dv[0]):
                assert perr == H.NOT_ENOUGH_DATA, (j, part, k, perr)
                rest[k] = chunks[k][cons:]
            n_calls += len(dv[1])
            ok += sum(c["error_code"] == 0 and c["grpc_status"] == 0 for c in dv[1])
    assert all(not r for r in rest.values())
    assert n_calls == n * n_sent and ok > n * 100


def test_mutated_server_streams_many_connections_per_batch():
    """The recorded conversation on n connections in lockstep; at one received segment each connection gets its own mutation of it
    (tests/_h2client_cases.mutate: frame head fields, payload bytes, cuts, repeated frames, hostile frames), then the conversation goes
    on: device == oracle call for call, connections that stopped with a parse error drop out."""
    import random
    from _h2client_cases import mutate
    cap, steps = _capture()
    recv_at = [j for j, s in enumerate(steps) if s[0] == "recv"]
    rng = random.Random(20261016)
    n = 48; n_calls = 0; n_errors = 0
    for j in recv_at[:6]:
        ctx = _ctx(n, cap["pending"], cap["stream_bytes"])
        dev = DeviceClients(ctx, range(n)); orc = OracleClients(n, cap["pending"], cap["stream_bytes"])
        rest = {k: b"" for k in range(n)}; ids = []
        for jj, st in enumerate(steps[:j + 3]):
            live = [k for k in range(n) if rest[k] is not None]
            if st[0] == "send":
                calls = [(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for k in live for p, b, e in st[1]]
                d = dev.pack(calls)
                assert d == orc.pack(calls), jj
                ids = sorted({sid for _, sid, _ in d})
                continue
            chunks = {k: rest[k] + (mutate(rng, st[1], ids) if jj == j else st[1]) for k in live}
            dv, ov = dev.parse(chunks, REGION, 128), orc.parse(chunks, REGION, 128)
            same(dv, ov, (j, jj))
            n_calls += len(dv[1])
            for k, (perr, cons, _) in zip(live, dv[0]):
                if perr == H.NOT_ENOUGH_DATA:
                    rest[k] = chunks[k][cons:]
                else:
                    rest[k] = None; n_errors += 1
    assert n_calls > 500 and n_errors > 5


def test_hand_built_frames_and_server_connections_in_the_same_batch():
    """Every hand-built case on a connection of its own, all in the same batches, next to server connections (b2_h2_conn_reset) whose
    requests go through b2_h2_process_batch unchanged; a client parse of a server connection reads nothing."""
    import _oracle as O
    from brpc_b200.abi import RUN_DT
    nc = len(HAND_CASES)
    ctx = _ctx(64, 8, STREAM_BYTES)
    dev = DeviceClients(ctx, range(nc)); orc = OracleClients(nc, 8, STREAM_BYTES)
    dchunks = [f(dev, k) for k, f in enumerate(HAND_CASES)]
    ochunks = [f(orc, k) for k, f in enumerate(HAND_CASES)]
    assert dchunks == ochunks
    servers = [40, 41]
    for s in servers:
        ctx.h2_conn_reset(s)
    srv_orc = {s: O.H2Conn() for s in servers}
    preface = b"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n" + bytes.fromhex("000000040000000000")
    n_calls = 0
    for step in range(max(len(c) for c in dchunks)):
        chunks = {k: c[step] for k, c in enumerate(dchunks) if step < len(c)}
        dv, ov = dev.parse(chunks, REGION, 64), orc.parse(chunks, REGION, 64)
        same(dv, ov, step)
        n_calls += len(dv[1])
        # the server connections: the client parser refuses them, the server parser sees them as before
        rs, _ = dev.parse({s: preface for s in servers}, REGION, 64)
        assert [r[:2] for r in rs] == [(H.TRY_OTHERS, 0)] * 2
        data = np.frombuffer(preface * 2, np.uint8); runs = np.zeros(2, RUN_DT)
        for i, s in enumerate(servers):
            runs[i]["offset"] = i * len(preface); runs[i]["length"] = len(preface); runs[i]["socket_id"] = s
        srs, msgs, out = ctx.h2_process_batch(data, runs)
        for i, s in enumerate(servers):
            err, cons, m, ctrl, _, _, _ = srv_orc[s].consume(preface)
            assert (int(srs[i]["parse_error"]), int(srs[i]["consumed"])) == (err, cons)
            assert out[int(srs[i]["ctrl_off"]):int(srs[i]["ctrl_off"]) + int(srs[i]["ctrl_len"])].tobytes() == ctrl
        servers_next = preface[24:]
        preface = servers_next                                                   # (later batches: a SETTINGS frame only)
    assert n_calls >= 20
    # refusals after the cases: GOAWAY (LOGOFF) and max_concurrent_streams (ELIMIT) on the connections those cases left behind
    calls = [(k, 1 | 8 | 16, ECHO, b"h:1", b"application/grpc", b"x", GRPC_EXTRA) for k in range(nc)]
    d, o = dev.pack(calls), orc.pack(calls)
    assert d == o and {st for st, _, _ in d} >= {H.REQ_OK, H.REQ_LOGOFF, H.REQ_ELIMIT}


def test_pool_exhaustion_both_ways():
    """NO_ROOM from b2_h2_pack_requests when the connection's stream records are taken, B2_PARSE_ERROR_NO_RESOURCE from the parser when a
    body outgrows its record or the calls outgrow call_cap — each the same as the oracle's model of the device."""
    from _h2client_cases import frame, grpc_body, OK_HDRS, trailers
    ctx = _ctx(8, 2, 69632)
    dev = DeviceClients(ctx, range(3)); orc = OracleClients(3, 2, 69632)
    calls = [(k, 1 | 8 | 16, ECHO, b"h:1", b"application/grpc", b"q", GRPC_EXTRA) for k in range(3) for _ in range(3)]
    d, o = dev.pack(calls), orc.pack(calls)
    assert d == o and [x[:2] for x in d[:3]] == [(0, 1), (0, 3), (H.REQ_NO_ROOM, 0)]
    big = frame(1, 4, 1, OK_HDRS) + b"".join(frame(0, 0, 1, b"b" * 16000) for _ in range(5))     # 80 000 bytes > 64 KiB of body room
    two = frame(1, 5, 1, OK_HDRS + trailers()) + frame(1, 5, 3, OK_HDRS + trailers())
    chunks = {0: big, 1: two, 2: frame(1, 4, 3, OK_HDRS) + frame(0, 1, 3, grpc_body(b"m" * 100))}
    dv, ov = dev.parse(chunks, REGION, 1), orc.parse(chunks, REGION, 1)
    same(dv, ov, "exhaustion")
    assert [r[0] for r in dv[0]] == [H.NO_RESOURCE, H.NO_RESOURCE, H.NOT_ENOUGH_DATA] and len(dv[1]) == 2
    # the freed records take new calls again
    calls = [(2, 1 | 8 | 16, ECHO, b"h:1", b"application/grpc", b"q", GRPC_EXTRA)]
    d, o = dev.pack(calls), orc.pack(calls)
    assert d == o and d[0][:2] == (H.REQ_OK, 5)


def test_live_round_trip_with_a_grpcio_server():
    """1000 calls over 8 connections: requests packed on the device, the server's frames parsed on the device, and only what the device
    wrote back (SETTINGS / PING acks, WINDOW_UPDATEs) sent to the server — bodies larger than the server's initial 65535-byte windows."""
    pytest.importorskip("grpc")
    srv, port = grpcio_server()
    ctx = _ctx(8, 128, (128 << 10) + 4096)
    dev = DeviceClients(ctx, range(8))
    n = 0
    try:
        for k in range(8):
            with socket.create_connection(("127.0.0.1", port)) as s:
                s.settimeout(60)
                batches = [[(ECHO, b"first", GRPC_EXTRA)]]            # the server's SETTINGS come back before large bodies go out, as
                for b in range(5):                                      # brpc sends with the maximised window until then (:326-339)
                    batch = []
                    for i in range(25):
                        q = k * 125 + b * 25 + i
                        size = [0, 7, 300, 4096, 20000, 70000][q % 6] if q % 5 else 100
                        path = ECHO if q % 17 else (ABORT if q % 2 else b"/example.Nope/Missing")
                        batch.append((path, bytes((q + j) & 0xff for j in range(size)), GRPC_EXTRA))
                    batches.append(batch)
                done = run_socket(dev, s, k, batches)
                sent = [c for b in batches for c in b]
                assert len(done) == len(sent)
                n -= 1
                for sid, (path, body, _) in zip(sorted(done), sent):
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
