"""Writes tests/golden/h2_client_rx_capture.json.gz: one h2 client connection to a real grpcio server (gRPC C-core), driven by the test
oracle's client (tests/_h2client_oracle.py: requests packed, the server's frames parsed, only the parser's own acks and WINDOW_UPDATEs
written back).  Recorded: every batch of calls with the bytes sent for it, and every chunk of bytes received, in order — so that device
tests replay the server's byte stream without depending on grpcio or its timing.  Run: python tests/golden/gen_h2_client_rx_capture.py"""
import gzip
import json
import os
import socket
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from _h2client_loop import ABORT, ECHO, GRPC_EXTRA, OracleClients, grpcio_server, run_socket  # noqa: E402

SIZES = [0, 1, 5, 100, 1000, 4096, 16379, 16384, 16385, 40000, 70000]
PENDING, STREAM_BYTES = 128, (128 << 10) + 4096


def body_of(i, n):
    return bytes((i * 7 + k) & 0xff for k in range(n))


def batches():
    one = [[(ECHO, body_of(i, n), GRPC_EXTRA + ((b"x-call", b"c%d" % i),))] for i, n in enumerate(SIZES)]
    burst = [[(ECHO if i % 9 else ABORT if i % 2 else b"/example.Nope/Missing", body_of(i, [0, 3, 100, 700][i % 4]),
               GRPC_EXTRA + ((b"x-call", b"b%d" % (i % 6)),)) for i in range(110)]]
    return one + burst + [[(ECHO, body_of(99, 70000), GRPC_EXTRA)]]


def main():
    srv, port = grpcio_server()
    rec = []
    try:
        cl = OracleClients(1, pending=PENDING, stream_bytes=STREAM_BYTES)
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(30)
            run_socket(cl, s, 0, batches(), record=rec)
    finally:
        srv.stop(0)
    events = []
    for e in rec:
        if e[0] == "send":
            events.append({"send": [[p.hex(), b.hex(), [[n.hex(), v.hex()] for n, v in ex]] for p, b, ex in e[1]], "wire_hex": e[2].hex()})
        else:
            events.append({"recv_hex": e[1].hex()})
    out = {"generator": "tests/golden/gen_h2_client_rx_capture.py", "server": "grpcio (gRPC C-core)", "pending": PENDING, "stream_bytes": STREAM_BYTES,
           "events": events}
    with gzip.open(os.path.join(HERE, "h2_client_rx_capture.json.gz"), "wt") as f:
        json.dump(out, f)
    print("%d events, %d received bytes" % (len(events), sum(len(e.get("recv_hex", "")) // 2 for e in events)))


if __name__ == "__main__":
    main()
