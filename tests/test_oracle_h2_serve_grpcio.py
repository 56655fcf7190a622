"""CPU: the serve oracle (tests/_h2serve.py) behind a TCP loop, against real gRPC C-core clients (grpcio) sending raw messages through
identity serializers: well-formed calls come back as EchoResponse, malformed ones as INVALID_ARGUMENT with brpc's error text after grpcio's
percent-decoding, and a gzip client on an opted-in connection is answered from the inflated bytes.  Also the pieces of the oracle that
brpc's sources fix outright: PercentEncode and the longest error text."""
import pytest

import _h2serve as S
import _oracle as O
from _h2loop import H2LoopServer

IDENTITY = b"127.0.0.1:8010"


def test_percent_encode_and_the_longest_error_text():
    assert S.percent_encode(b"[E1003]Invalid gRPC request") == b"%5bE%31%30%30%33%5dInvalid%20gRPC%20request"
    assert S.percent_encode(bytes(range(256))).count(b"%") == 256 - 26 - 26 - 4
    rt = b"x" * 95                                               # b2_register_method keeps request_type_name below 96 bytes
    text = S.error_text(b"9" * 63, S.reason_empty(rt))          # and b2_set_server_identity the identity below 64
    assert len(text) == 234 and len(S.percent_encode(text)) <= 702


def _serve(engine, requests, channels, compression=None):
    srv = H2LoopServer(engine)
    try:
        got = S.grpcio_calls(srv.port, requests, channels=channels, compression=compression)
    finally:
        srv.close()
    assert not srv.errors, srv.errors
    return got


def test_grpcio_client_gets_echo_replies_and_brpc_error_texts():
    pytest.importorskip("grpc")
    reqs = S.mutation_corpus(360)
    eng = S.OracleServeEngine(identity=IDENTITY)
    got = _serve(eng, reqs, channels=4)
    codes = set()
    for i, (raw, g) in enumerate(zip(reqs, got)):
        assert g == S.expected_call(raw, IDENTITY), (i, raw[:16], g[:2])
        codes.add(g[0])
    assert codes == {"OK", "INVALID_ARGUMENT"} and eng.n_answered == len(reqs) and 100 < eng.n_errors < 200
    assert got[0][1] == "[127.0.0.1:8010][E1003]Fail to parse http body as example.EchoRequest"


def test_grpcio_gzip_client_is_answered_from_the_inflated_bytes():
    pytest.importorskip("grpc")
    import grpc
    reqs = [S.echo_request((b"compressible text %d; " % i) * (i % 50 + 1)) for i in range(200)]
    eng = S.OracleServeEngine(gunzip=True)
    got = _serve(eng, reqs, channels=2, compression=grpc.Compression.Gzip)
    assert got == [("OK", "", r) for r in reqs]
    assert eng.n_inflated > 100 and eng.n_answered == len(reqs)


def test_other_methods_and_unknown_paths_are_left_to_the_host():
    """a B2_HANDLER_HOST method, a gzip-replying echo method and an unknown path: none answered (the host's UNIMPLEMENTED comes back)"""
    pytest.importorskip("grpc")
    import grpc
    methods = (O.ECHO_METHOD, dict(O.ECHO_METHOD, method_name=b"Host", handler=0), dict(O.ECHO_METHOD, method_name=b"Gz", response_compress_type=2))
    eng = S.OracleServeEngine(methods=methods)
    srv = H2LoopServer(eng)
    try:
        ch = grpc.insecure_channel("127.0.0.1:%d" % srv.port)
        for path in (b"/example.EchoService/Host", b"/example.EchoService/Gz", b"/other.Service/Echo"):
            call = ch.unary_unary(path.decode(), request_serializer=lambda b: b, response_deserializer=lambda b: b)
            with pytest.raises(grpc.RpcError) as e:
                call(S.echo_request(b"hi"), timeout=30)
            assert e.value.code() == grpc.StatusCode.UNIMPLEMENTED
        call = ch.unary_unary("/example.EchoService/Echo", request_serializer=lambda b: b, response_deserializer=lambda b: b)
        assert call(S.echo_request(b"hi"), timeout=30) == S.echo_request(b"hi")
        ch.close()
    finally:
        srv.close()
    assert eng.n_answered == 1 and not srv.errors
