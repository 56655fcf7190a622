"""CPU: the gunzip oracle (tests/_h2gzip.py) against real gRPC C-core (grpcio with compression=Gzip), both directions, and the listed
deviation of the device's one-block model pinned against the system zlib:
  * a gzip grpcio SERVER answering the oracle client: every inflated reply equals what was sent, small replies sent uncompressed under
    grpc-encoding: gzip are left alone;
  * a gzip grpcio CLIENT against a TCP loop whose engine is the C oracle with the gunzip step, echoing the inflated request: every call
    returns its request;
  * policy::GzipDecompressBase restated over a list of IOBuf blocks: with ONE block it never fails and hands over exactly what the device
    models (_gzipstream), over the whole mutation corpus; with several blocks it sometimes fails ("Fail to un-gzip"), depending on where
    the blocks end — the reason the device, which takes a message as one block, never does.
Both live parts assert that compressed messages actually occurred."""
import random
import socket
import zlib

import pytest

import _gzipstream as Z
import _h2client_oracle as H
import _h2gzip as G
from _h2client_loop import ECHO, GRPC_EXTRA, OracleClients, run_socket


class GzOracleClients(OracleClients):
    def __init__(self, n, pending, stream_bytes):
        self.c = [G.GzClientConn(pending, stream_bytes, gunzip=True) for _ in range(n)]


def test_oracle_client_against_a_gzip_grpcio_server():
    pytest.importorskip("grpc")
    srv, port = G.gzip_grpcio_server()
    bodies = G.echo_bodies(210)
    try:
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(60)
            batches = [[(ECHO, b"first", GRPC_EXTRA)]] + [[(ECHO, b, GRPC_EXTRA) for b in bodies[i:i + 30]] for i in range(0, len(bodies), 30)]
            done = run_socket(GzOracleClients(1, 64, (128 << 10) + 4096), s, 0, batches)
    finally:
        srv.stop(0)
    sent = [b for bt in batches for _, b, _ in bt]
    assert len(done) == len(sent)
    n_gz = n_plain_under_gzip = 0
    for sid, body in zip(sorted(done), sent):
        c = done[sid]
        assert c["error_code"] == 0 and c["msg"] == body, (sid, len(body))
        enc = H.get(c["headers"], b"grpc-encoding")
        if c["flags"] & G.F_GUNZIPPED:
            assert c["flags"] & H.F_COMPRESSED and enc == b"gzip"; n_gz += 1
        elif enc == b"gzip":
            assert not c["flags"] & H.F_COMPRESSED; n_plain_under_gzip += 1
    assert n_gz > 80 and n_plain_under_gzip > 20, (n_gz, n_plain_under_gzip)


def test_gzip_grpcio_client_against_the_oracle_echo_server():
    pytest.importorskip("grpc")
    from _h2loop import H2LoopServer
    eng = G.OracleGzEngine()
    srv = H2LoopServer(eng)
    bodies = G.echo_bodies(300, seed=6)
    try:
        got = G.grpcio_gzip_client_calls(srv.port, bodies, in_flight=64)
    finally:
        srv.close()
    assert got == bodies and not srv.errors, srv.errors
    assert eng.n_compressed > 100, eng.n_compressed


def corpus(rng):
    seeds = [_gz(p, lv, st) for p in (b"corpus text %d " * 900, bytes(rng.randrange(256) for _ in range(70000)), b"\3" * 200000)
             for lv, st in ((6, zlib.Z_DEFAULT_STRATEGY), (0, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED))]
    out = list(seeds)
    for _ in range(300):
        b = bytearray(rng.choice(seeds)); k = rng.random()
        if k < 0.5:
            b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        elif k < 0.75:
            b = b[:rng.randrange(len(b))]
        else:
            b += b"trailing garbage"
        out.append(bytes(b))
    return out


def _gz(data, level, strategy):
    c = zlib.compressobj(level, zlib.DEFLATED, 31, 9, strategy)
    return c.compress(data) + c.flush()


def test_gzip_decompress_base_one_block_never_fails_several_blocks_sometimes_do():
    rng = random.Random(11)
    n_fail = 0; n_valid = 0
    for s in corpus(rng):
        ok, got = G.gzip_decompress_base([s])
        assert ok and got == Z.gzip_input_stream(s, Z.GZIP)              # the device's model: one block
        cuts = sorted(rng.sample(range(1, len(s)), min(len(s) - 1, rng.randrange(1, 5)))) if len(s) > 1 else []
        blocks = [s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])]
        ok_n, got_n = G.gzip_decompress_base(blocks)
        valid = zlib.decompressobj(31)
        try:
            whole = valid.decompress(s); complete = valid.eof and not valid.unused_data
        except zlib.error:
            complete = False
        if complete:
            n_valid += 1
            assert ok_n and got_n == whole                               # an intact stream never fails, whatever the blocks
        n_fail += not ok_n
    assert n_valid >= 9 and n_fail > 20, (n_valid, n_fail)
