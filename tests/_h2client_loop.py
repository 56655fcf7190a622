"""Test helpers for the receiving half of h2 client connections: the same interface over the oracle (_h2client_oracle.ClientConn) and the
device (b2_h2_pack_requests + b2_h2_client_process_batch), the normalised form of a b2_h2_call, and a client loop against a socket that
answers the server only with what the parser itself wrote back (no host-side mirroring)."""
import numpy as np

import _h2client_oracle as H
import _oracle as O

GRPC_EXTRA = ((b"te", b"trailers"), (b"grpc-accept-encoding", b"identity,gzip"))
ECHO = b"/example.EchoService/Echo"
ABORT = b"/example.EchoService/Abort"
ABORT_TEXT = "bad thing: 100% wrong, \u00fcn\u00efcode\n2nd line"                 # grpc-message needs percent-encoding


def grpcio_server():
    """A gRPC C-core server: Echo echoes, Abort fails with FAILED_PRECONDITION and ABORT_TEXT, anything else is UNIMPLEMENTED."""
    from concurrent import futures
    import grpc

    class Handler(grpc.GenericRpcHandler):
        def service(self, details):
            ident = dict(request_deserializer=lambda b: b, response_serializer=lambda b: b)
            if details.method == ECHO.decode():
                return grpc.unary_unary_rpc_method_handler(lambda req, ctx: req, **ident)
            if details.method == ABORT.decode():
                def abort(req, ctx):
                    ctx.abort(grpc.StatusCode.FAILED_PRECONDITION, ABORT_TEXT)
                return grpc.unary_unary_rpc_method_handler(abort, **ident)
            return None
    srv = grpc.server(futures.ThreadPoolExecutor(max_workers=16), handlers=[Handler()],
                      options=[("grpc.max_receive_message_length", 1 << 24), ("grpc.max_send_message_length", 1 << 24)])
    port = srv.add_insecure_port("127.0.0.1:0")
    srv.start()
    return srv, port


def records(buf):
    out = []; p = 0
    while p < len(buf):
        nl = buf[p] | (buf[p + 1] << 8); vl = buf[p + 2] | (buf[p + 3] << 8)
        out.append((bytes(buf[p + 4:p + 4 + nl]), bytes(buf[p + 4 + nl:p + 4 + nl + vl]))); p += 4 + nl + vl
    return out


def norm_oracle(c):
    return dict(run_idx=c["run_idx"], stream_id=c["stream_id"], how=c["how"], status_code=c["status_code"], error_code=c["error_code"],
                grpc_status=c["grpc_status"], flags=c["flags"], headers=c["headers"], body=c["body"], msg=c["msg"], error=c["error"],
                headers_off=c["headers_off"], body_off=c["body_off"], msg_off=c["msg_off"], error_off=c["error_off"])


def norm_device(c, out, inp):
    src = inp if c["flags"] & H.F_BODY_IN_INPUT else out
    g = lambda buf, off, n: bytes(buf[int(off):int(off) + int(n)])
    return dict(run_idx=int(c["run_idx"]), stream_id=int(c["stream_id"]), how=int(c["how"]), status_code=int(c["status_code"]),
                error_code=int(c["error_code"]), grpc_status=int(c["grpc_status"]), flags=int(c["flags"]),
                headers=records(g(out, c["headers_off"], c["headers_len"])), body=g(src, c["body_off"], c["body_len"]),
                msg=g(src, c["msg_off"], c["msg_len"]), error=g(out, c["error_off"], c["error_len"]),
                headers_off=int(c["headers_off"]), body_off=int(c["body_off"]), msg_off=int(c["msg_off"]), error_off=int(c["error_off"]))


class OracleClients:
    """n oracle client connections; batch calls look like the device's"""
    def __init__(self, n, pending=8, stream_bytes=69632):
        self.c = [H.ClientConn(pending, stream_bytes) for _ in range(n)]

    def pack(self, calls):
        """calls: (conn, flags, path, authority, content_type, body, extra) -> [(status, stream_id, bytes)]"""
        return [self.c[k].pack_request(p, a, b, content_type=ct, flags=f, extra=e) for k, f, p, a, ct, b, e in calls]

    def parse(self, chunks, region, call_cap):
        """chunks: {conn: bytes}, one run each in dict order -> ([(parse_error, consumed, ctrl)], [normalised calls])"""
        data = b"".join(chunks.values()); runs = []; off = 0; calls = []
        for r, (k, b) in enumerate(chunks.items()):
            perr, cons, cl, ctrl, _ = self.c[k].consume(data, off, len(b), r, region, call_cap)
            runs.append((perr, cons, ctrl)); calls += [norm_oracle(x) for x in cl]
            off += len(b)
        return runs, calls

    def abandon(self, conn, ids):
        self.c[conn].abandon(ids)


class DeviceClients:
    def __init__(self, ctx, conns):
        self.ctx = ctx
        for k in conns:
            ctx.h2_client_conn_reset(k)

    def pack(self, calls):
        from brpc_b200.abi import H2_REQUEST_DT
        blob, reqs = O.h2_request_blob(calls)
        out_cap = sum(1024 + len(c[5]) + len(c[5]) // 1000 for c in calls) + 4096           # (what b2_h2_pack_requests reserves per request)
        res, got = self.ctx.h2_pack_requests(np.frombuffer(blob, np.uint8), reqs.astype(H2_REQUEST_DT), out_cap=out_cap)
        return [(int(r["status"]), int(r["stream_id"]), g) for r, g in zip(res, got)]

    def parse(self, chunks, region, call_cap):
        from brpc_b200.abi import RUN_DT
        data = np.frombuffer(b"".join(chunks.values()) + b"\0", np.uint8)
        runs = np.zeros(len(chunks), RUN_DT); off = 0
        for r, (k, b) in enumerate(chunks.items()):
            runs[r]["offset"] = off; runs[r]["length"] = len(b); runs[r]["socket_id"] = k; off += len(b)
        rs, calls, out = self.ctx.h2_client_process_batch(data, runs, call_cap=call_cap * len(chunks), out_cap=region * len(chunks))
        res = [(int(s["parse_error"]), int(s["consumed"]), out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()) for s in rs]
        return res, [norm_device(c, out, data) for c in calls]

    def abandon(self, conn, ids):
        self.ctx.h2_client_abandon_streams(conn, ids)


def run_socket(client, sock, conn, batches, region=1 << 22, call_cap=512, record=None, timeout_rounds=20000):
    """Sends each batch of calls (path, body, extra) on connection `conn`, then reads until every sent stream has left the connection.
    The server's bytes go to the parser as they arrive; only the parser's own ctrl bytes are written back.  Returns {stream: call}."""
    done = {}; pending = b""
    for batch in batches:
        calls = [(conn, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for p, b, e in batch]
        res = client.pack(calls)
        sent = []
        for st, sid, b in res:
            assert st == 0, (st, sid)
            sent.append(sid)
        wire = b"".join(b for _, _, b in res)
        sock.sendall(wire)
        if record is not None:
            record.append(("send", [(p, b, e) for p, b, e in batch], wire))
        rounds = 0
        while not all(s in done for s in sent):
            d = sock.recv(1 << 16)
            assert d, "server closed the connection"
            if record is not None:
                record.append(("recv", d))
            pending += d
            runs, got = client.parse({conn: pending}, region, call_cap)
            perr, cons, ctrl = runs[0]
            pending = pending[cons:]
            if ctrl:
                sock.sendall(ctrl)
            rounds += 1
            assert rounds < timeout_rounds and perr == H.NOT_ENOUGH_DATA, (perr, rounds)
            for c in got:
                done[c["stream_id"]] = c
    return done
