"""CPU: pins the oracle of the RECEIVING half of an h2 client connection (tests/_h2client_oracle.py: ParseH2Message on a connected socket,
OnEndStream / OnResetStream / OnGoAway, ProcessHttpResponse's verdict) against an independent server — a real grpcio server (gRPC C-core):
its SETTINGS, SETTINGS ACK, PINGs, WINDOW_UPDATEs, HEADERS with its own HPACK dynamic table, DATA and trailers go into the oracle's
parser, and only what the parser writes back (acks, WINDOW_UPDATEs) is sent to the server — nothing is mirrored by the host.  Then the
same oracle on hand-built frames for what a well-behaved server does not send."""
from concurrent import futures
import socket

import pytest

import _h2client_oracle as H
from _h2client_cases import HAND_CASES, STREAM_BYTES, grpc_body
from _h2client_loop import ABORT_TEXT, ECHO, GRPC_EXTRA, OracleClients, grpcio_server, run_socket

grpc = pytest.importorskip("grpc")

SIZES = [0, 1, 5, 100, 1000, 4096, 16379, 16384, 16385, 40000, 65536, 70000, 200000]


def body_of(i, n):
    return bytes((i * 7 + k) & 0xff for k in range(n))


def check_calls(done, batches):
    n = 0
    for sid, (path, body, _) in zip(sorted(done), [c for b in batches for c in b]):
        c = done[sid]
        assert c["how"] == H.ENDED and c["status_code"] == 200, c
        hdr = dict(c["headers"])
        assert hdr[b"content-type"] == b"application/grpc"
        if path == ECHO:
            assert c["error_code"] == 0 and c["grpc_status"] == 0 and c["msg"] == body and c["flags"] & H.F_PREFIX_OK, (sid, len(body))
        elif path.endswith(b"/Abort"):
            assert (c["grpc_status"], c["error_code"]) == (9, 2001) and c["error"] == ABORT_TEXT.encode(), c["error"]   # FAILED_PRECONDITION -> EINTERNAL
        else:
            assert (c["grpc_status"], c["error_code"]) == (12, 1002), c                                                 # UNIMPLEMENTED -> ENOMETHOD
        n += 1
    return n


def test_oracle_client_parser_against_a_grpcio_server():
    srv, port = grpcio_server()
    try:
        cl = OracleClients(1, pending=256, stream_bytes=(256 << 10) + 4096)
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(30)
            one = [[(ECHO, body_of(i, n), GRPC_EXTRA + ((b"x-call", b"c%d" % i),))] for i, n in enumerate(SIZES)]
            burst = [[(ECHO if i % 9 else b"/example.EchoService/Abort" if i % 2 else b"/example.Nope/Missing", body_of(i, SIZES[i % 8]),
                       GRPC_EXTRA) for i in range(120)]]
            batches = one + burst
            done = run_socket(cl, s, 0, batches)
        assert check_calls(done, batches) == len(SIZES) + 120
        conn = cl.c[0]
        assert not conn.streams and conn.settings_received and conn.hp is not None
    finally:
        srv.stop(0)


def _run_case(f):
    cl = OracleClients(1, pending=8, stream_bytes=STREAM_BYTES)
    out = []
    for ch in f(cl, 0):
        runs, calls = cl.parse({0: ch}, 1 << 20, 64)
        out.append((runs[0], calls))
    return cl, out


def test_oracle_client_parser_on_hand_built_frames():
    by = {f.__name__: _run_case(f) for f in HAND_CASES}
    (_, calls), = by["case_unary_ok_and_trailers_merge"][1]
    c, = calls
    assert dict(c["headers"]) == {b"content-type": b"application/grpc+proto", b"x-dup": b"a,b", b"cookie": b"k=1; k=2", b"x-empty": b"z",
                                  b"set-cookie": b"s=2", b"grpc-status": b"0"}
    assert [v for n, v in c["headers"] if n == b"set-cookie"] == [b"s=1", b"s=2"] and c["msg"] == b"hello" and c["error_code"] == 0
    (run, calls), = by["case_rst_stream_from_peer_and_unknown"][1]
    assert [(c["how"], c["status_code"]) for c in calls] == [(H.RESET_BY_PEER, 503), (H.RESET_BY_PEER, 503)]
    assert run[2].endswith(bytes([0, 0, 8, 7, 0, 0, 0, 0, 0, 0xff, 0xff, 0xff, 0xff, 0, 0, 0, 6]))     # GOAWAY(FRAME_SIZE_ERROR)
    cl, ((run, calls),) = by["case_goaway_above_and_below"]
    assert [(c["stream_id"], c["how"], c["status_code"]) for c in calls] == [(1, 0, 200), (7, 3, 503), (9, 3, 503), (11, 3, 503), (3, 0, 200)]
    assert calls[-1]["error_code"] == 2001 and cl.c[0].goaway == 5
    st, sid, b = cl.c[0].pack_request(ECHO, b"h:1", b"x")
    assert (st, sid, b) == (H.REQ_LOGOFF, 13, b"")
    (_, calls), = by["case_goaway_zero_takes_all"][1]
    assert [c["stream_id"] for c in calls] == [1, 3, 5, 7, 9] and calls[3]["body"] == grpc_body(b"partial")
    (_, calls), = by["case_headers_on_unknown_streams_advance_hpack"][1]
    assert [h for h in calls[0]["headers"] if h[0].startswith(b"x-")] == [(b"x-cont", b"v3"), (b"x-more", b"v2"), (b"x-table", b"v1")]
    (run, calls), = by["case_bad_status_and_unknown_pseudo"][1]
    # ":status: 20x" fails ConsumeHeaders: GOAWAY(PROTOCOL_ERROR), and the rest of that payload is read as the next frame head
    assert calls == [] and run[2] == bytes([0, 0, 8, 7, 0, 0, 0, 0, 0, 0xff, 0xff, 0xff, 0xff, 0, 0, 0, 1]) and run[1] == 9
    (_, calls), = by["case_grpc_prefix_missing_short_and_compressed"][1]
    assert [(c["error_code"], c["error"]) for c in calls] == [(2002, b"Invalid gRPC response")] * 2 + \
        [(2002, b"Fail to find header `grpc-encoding' in compressed gRPC response"), (0, b"")]
    assert calls[3]["flags"] & H.F_COMPRESSED and calls[3]["msg"] == b"zz"
    (_, calls), = by["case_non_2xx_with_long_body_and_percent_message"][1]
    assert calls[0]["error_code"] == 1010 and calls[0]["error"].startswith(b"HTTP/2.0 404 Not Found: ABCD") and len(calls[0]["error"]) == 24 + 2048
    assert calls[1]["error"] == b"HTTP/2.0 418 Unknown status code (418)"
    assert calls[2]["error"] == b"down for maint\xe2\x9c\x93%" and calls[2]["error_code"] == 2001
    assert calls[3]["error"] == b"GRPC_INVALIDARGUMENT" and calls[3]["error_code"] == 22
    cl, ((run, calls),) = by["case_settings_ack_ping_window_update"]
    assert run[2].startswith(b"\0\0\0\x04\x01\0\0\0\0" + b"\0\0\x08\x06\x01\0\0\0\0" + b"12345678")
    conn = cl.c[0]
    assert conn.r["mcs"] == 2 and conn.r["sws"] == 1 << 20 and conn.window == 65535 - 4 * 6 + 1000
    assert [cl.c[0].pack_request(ECHO, b"h:1", b"x")[0] for _ in range(2)] == [H.REQ_ELIMIT, H.REQ_ELIMIT]   # 4 pending > 2
    cl, ((run0, c0), (run1, c1)) = by["case_data_on_unknown_stream_and_window_updates"]
    assert run0[2].startswith(bytes([0, 0, 4, 3, 0, 0, 0, 0x03, 0xe9, 0, 0, 0, 5]))    # RST_STREAM(STREAM_CLOSED) for 1001
    assert c1 == [] and run1[2].count(bytes([0, 0, 4, 8, 0, 0, 0, 0, 1])) == 4 and run1[0] == H.NOT_ENOUGH_DATA                   # the stream's quota came back as WINDOW_UPDATEs
    cl, ((run0, c0), (run1, c1)) = by["case_abandoned_streams"]
    assert [c["stream_id"] for c in c0] == [1] and not c1 and set(cl.c[0].streams) == {7}
    cl, ((run0, c0), (run1, c1)) = by["case_goaway_last_stream_id_with_the_high_bit"]
    assert [(c["stream_id"], c["how"], c["status_code"]) for c in c0] == [(1, 3, 503), (3, 3, 503)] and c1 == [] and not cl.c[0].streams
    assert cl.c[0].goaway == -(1 << 31) and cl.c[0].pack_request(ECHO, b"h:1", b"x")[:2] == (H.REQ_OK, 5)
    cl, ((run0, c0),) = by["case_abandoned_stream_completing_first_is_reported"]
    assert [c["stream_id"] for c in c0] == [1, 3] and set(cl.c[0].streams) == {7}
    # the device's stream pool: NO_ROOM without consuming an id
    cl = OracleClients(1, pending=2)
    res = cl.pack([(0, 1 | 8 | 16, ECHO, b"h:1", b"application/grpc", b"q", GRPC_EXTRA) for _ in range(3)])
    assert [(s, i) for s, i, _ in res] == [(0, 1), (0, 3), (H.REQ_NO_ROOM, 0)]
