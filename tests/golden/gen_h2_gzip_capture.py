"""Writes tests/golden/h2_gzip_capture.json.gz: both directions of gRPC C-core's gzip compression (grpcio, compression=Gzip), so that the
device tests of the gunzip step replay fixed bytes instead of depending on grpcio's timing.
  - "client_rx": the oracle client (tests/_h2gzip.GzClientConn) calling a gzip grpcio SERVER: what was sent and every chunk received, in
    order (the events of tests/_h2client_loop.run_socket, as in gen_h2_client_rx_capture.py);
  - "server_rx": a gzip grpcio CLIENT calling a TCP loop whose engine is the C oracle with the gunzip step: every chunk the server
    received, per connection, in order, and the bodies of the calls.
    python tests/golden/gen_h2_gzip_capture.py"""
import gzip
import json
import os
import socket
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _h2gzip as G  # noqa: E402
from _h2client_loop import ECHO, GRPC_EXTRA, OracleClients, run_socket  # noqa: E402
from _h2loop import H2LoopServer  # noqa: E402

PENDING, STREAM_BYTES = 48, (128 << 10) + 4096


def bodies(n, seed):
    """text a gzip peer compresses (up to 20 KB) and small random bodies it sends as they are; kept small so the file stays small"""
    import random
    rng = random.Random(seed)
    return [bytes(rng.randrange(256) for _ in range([0, 40, 300][i % 3])) if i % 4 == 3 else
            (b"capture %d / %d; " % (i, seed) * 2000)[:[0, 3, 100, 600, 4096, 20000][i % 6]] for i in range(n)]


class _Clients(OracleClients):
    def __init__(self):
        self.c = [G.GzClientConn(PENDING, STREAM_BYTES, gunzip=True)]


def main():
    srv, port = G.gzip_grpcio_server()
    rec = []
    cbodies = bodies(80, 21)
    batches = [[(ECHO, b"first", GRPC_EXTRA)]] + [[(ECHO, b, GRPC_EXTRA) for b in cbodies[i:i + 40]] for i in range(0, len(cbodies), 40)]
    try:
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(60)
            run_socket(_Clients(), s, 0, batches, record=rec)
    finally:
        srv.stop(0)
    events = []
    for kind, x, *rest in rec:
        if kind == "send":
            events.append({"send": [(p.hex(), b.hex(), [(n.hex(), v.hex()) for n, v in e]) for p, b, e in x], "wire_hex": rest[0].hex()})
        else:
            events.append({"recv_hex": x.hex()})
    loop = H2LoopServer(G.OracleGzEngine())
    sbodies = bodies(100, 22)
    try:
        assert G.grpcio_gzip_client_calls(loop.port, sbodies, in_flight=32) == sbodies
    finally:
        loop.close()
    cap = {"pending": PENDING, "stream_bytes": STREAM_BYTES, "client_rx": events,
           "server_rx": {"bodies": [b.hex() for b in sbodies], "chunks": {str(k): [c.hex() for c in v] for k, v in loop.capture.items()}}}
    with gzip.open(os.path.join(HERE, "h2_gzip_capture.json.gz"), "wt") as f:
        json.dump(cap, f)


if __name__ == "__main__":
    main()
