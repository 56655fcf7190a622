"""Test oracle of the gunzip step on h2 / gRPC connections opted in with b2_h2_conn_set_gunzip: what ProcessHttpRequest
(src/brpc/policy/http_rpc_protocol.cpp:1645-1683) and ProcessHttpResponse (:507-529) do between RemoveGrpcPrefix and the protobuf parse,
with the device's placement of the inflated bytes, so that msg_off compares too.

  - the encoding: gRPC -> merged "grpc-encoding" only when the prefix says compressed (absent, on a call no earlier verdict failed:
    B2_H2_FLAG_NO_GRPC_ENCODING), other
    messages -> merged "content-encoding"; it must be exactly b"gzip";
  - candidates: server messages with a valid prefix or, not gRPC, a non-empty body; client calls with error_code 0;
  - GzipDecompress over ONE block: the bytes the system zlib hands over through GzipInputStream (_gzipstream), which cannot fail;
  - the device's bound (the C oracle's orc_gzip_sizing_bound, the model of gz_input_stream<false>), > 1 MiB in or out -> GUNZIP_HOST;
  - placement: 16-byte aligned after the run's parse bytes (region / 4 + blob_used), in message order, skipped (GUNZIP_HOST) when the
    bound does not fit before the region's end.
The client side is ClientConn of _h2client_oracle with the step at the end of each run; the server side applies it to the C oracle's
messages (whose records are raw: they are merged first, with the client oracle's merge)."""
import ctypes as C

import _gzipstream as Z
import _h2client_oracle as H
import _oracle as O

F_GUNZIPPED, F_GUNZIP_HOST, F_NO_GRPC_ENCODING = 64, 128, 256
GZ_MAX = 1 << 20                                                  # kGzMaxIn / kGzMaxOut

O.lib.orc_gzip_sizing_bound.restype = C.c_size_t
O.lib.orc_gzip_sizing_bound.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_size_t]


def sizing_bound(src):
    return O.lib.orc_gzip_sizing_bound(bytes(src), len(src), Z.GZIP, GZ_MAX)


def a16(n):
    return (n + 15) & ~15


def step(items, r, region, blob_used, client):
    """items: one dict per message of the run, in order: grpc, prefix_ok, compressed, merged (records), body, failed (a client call with an
    error), stopped (a client call an earlier verdict failed before the grpc-encoding check).
    Returns ([(flags to add, msg_off or None, inflated bytes or None)], new blob_used)."""
    cur = region // 4 + blob_used
    res = []
    for it in items:
        add = 0
        if it["grpc"]:
            if not (it["prefix_ok"] and it["compressed"]):
                res.append((0, None, None)); continue
            enc = H.get(it["merged"], b"grpc-encoding")
            if enc is None:
                res.append((0 if it.get("stopped") else F_NO_GRPC_ENCODING, None, None)); continue
        else:
            if not client and not it["body"]:
                res.append((0, None, None)); continue
            enc = H.get(it["merged"], b"content-encoding")
        if enc is None or it["failed"] or enc != b"gzip":
            res.append((add, None, None)); continue
        src = it["body"][5:] if it["grpc"] else it["body"]
        bound = sizing_bound(src) if len(src) <= GZ_MAX else GZ_MAX + 1
        if bound > GZ_MAX or cur + bound > region:
            res.append((F_GUNZIP_HOST, None, None)); continue
        got = Z.gzip_input_stream(src, Z.GZIP)
        assert len(got) <= bound, (len(got), bound)
        res.append((F_GUNZIPPED, r * region + cur, got))
        cur += a16(bound)
    return res, cur - region // 4


def apply_to_calls(calls, r, region, blob_used):
    """the step over the normalised oracle calls of one client run (in place); returns the new blob_used"""
    items = [dict(grpc=bool(c["flags"] & H.F_GRPC), prefix_ok=bool(c["flags"] & H.F_PREFIX_OK), compressed=bool(c["flags"] & H.F_COMPRESSED),
                  merged=c["headers"], body=c["body"], failed=c["error_code"] != 0,
                  stopped=c["error_code"] not in (0, 2002)) for c in calls]            # (2002 with a valid prefix: the grpc-encoding check itself)
    res, used = step(items, r, region, blob_used, True)
    for c, (add, off, got) in zip(calls, res):
        c["flags"] |= add
        if off is not None:
            c["msg_off"] = off; c["msg"] = got
    return used


class GzClientConn(H.ClientConn):
    """ClientConn with b2_h2_conn_set_gunzip(enable) on the connection"""
    def __init__(self, pending=8, stream_bytes=69632, gunzip=False):
        super().__init__(pending, stream_bytes)
        self.gunzip = gunzip

    def consume(self, data, run_off, run_len, r, region, call_cap):
        perr, cons, calls, ctrl, used = super().consume(data, run_off, run_len, r, region, call_cap)
        if self.gunzip:
            used = apply_to_calls(calls, r, region, used)
        return perr, cons, calls, ctrl, used


def server_step(msgs, blob, in_input, r, region, blob_used):
    """The step over the C oracle's messages of one server run (msgs: H2_MSG_DT records with offsets into blob).  in_input[i]: whether
    the device references message i's body in the input (B2_H2_FLAG_BODY_IN_INPUT).  Returns [(flags to add, msg_off, bytes)], blob_used."""
    from _h2client_loop import records
    items = []
    for m in msgs:
        f = int(m["flags"])
        hdr = bytes(blob[int(m["headers_off"]):int(m["headers_off"]) + int(m["headers_len"])])
        merged, _ = H.merge_headers(records(hdr))
        items.append(dict(grpc=bool(f & 1), prefix_ok=bool(f & 2), compressed=bool(f & 4), merged=merged,
                          body=bytes(blob[int(m["body_off"]):int(m["body_off"]) + int(m["body_len"])]), failed=False))
    return step(items, r, region, blob_used, False)


def server_blob_used(dev_msgs, r, region):
    """the bytes the device's parse wrote after region / 4 in run r: header records then, unless the body stays in the input, the body,
    each 16-byte aligned, message after message"""
    end = region // 4
    for m in dev_msgs:
        e = int(m["headers_off"]) - r * region + a16(int(m["headers_len"]))
        if not int(m["flags"]) & H.F_BODY_IN_INPUT:
            e += a16(int(m["body_len"]))
        end = max(end, e)
    return end - region // 4


def gzip_grpcio_server():
    """A gRPC C-core server configured with compression=Gzip whose Echo method echoes: it compresses every reply the client accepts gzip
    for (the client oracle's requests carry grpc-accept-encoding: identity,gzip) unless compressing does not make it smaller."""
    from concurrent import futures
    import grpc
    from _h2client_loop import ECHO

    class Handler(grpc.GenericRpcHandler):
        def service(self, details):
            if details.method == ECHO.decode():
                return grpc.unary_unary_rpc_method_handler(lambda req, ctx: req, request_deserializer=lambda b: b, response_serializer=lambda b: b)
            return None
    srv = grpc.server(futures.ThreadPoolExecutor(max_workers=8), handlers=[Handler()], compression=grpc.Compression.Gzip,
                      options=[("grpc.max_receive_message_length", 1 << 24), ("grpc.max_send_message_length", 1 << 24)])
    port = srv.add_insecure_port("127.0.0.1:0")
    srv.start()
    return srv, port


def gzip_decompress_base(blocks, fmt=Z.GZIP):
    """policy::GzipDecompressBase (src/brpc/policy/gzip_compress.cpp:138-176) over an IOBuf of `blocks`, on the system zlib: the
    GzipInputStream of _gzipstream with a sub-stream that hands out one block per Next().  Returns (ok, bytes copied out): it fails when
    the wrapper's ByteCount() falls short of the data (the stream ended in an error before the last block was fetched) or a further Next()
    succeeds."""
    zs = Z.ZStream()
    bufs = [C.create_string_buffer(b, len(b)) for b in blocks]
    outbuf = C.create_string_buffer(Z.K_BUFFER)
    out_base = C.addressof(outbuf)
    fetched = [0]                                                # IOBufAsZeroCopyInputStream::ByteCount (no BackUp is ever called)
    st = {"zerror": Z.Z_OK, "output_position": out_base, "next_block": 0}
    zs.next_out = out_base; zs.avail_out = Z.K_BUFFER
    got = bytearray()

    def sub_next():
        while st["next_block"] < len(blocks):                    # (IOBuf has no empty blocks)
            i = st["next_block"]; st["next_block"] += 1
            if len(blocks[i]):
                fetched[0] += len(blocks[i])
                return C.addressof(bufs[i]), len(blocks[i])
        return None

    def inflate_call():
        if st["zerror"] == Z.Z_OK and zs.avail_out == 0:
            pass
        elif zs.avail_in == 0:
            first = not zs.next_in
            nxt = sub_next()
            if nxt is None:
                zs.next_out = None; zs.avail_out = 0
                return Z.Z_STREAM_END
            zs.next_in, zs.avail_in = nxt
            if first:
                e = Z._init(zs, fmt)
                if e != Z.Z_OK:
                    return e
        zs.next_out = out_base; zs.avail_out = Z.K_BUFFER
        st["output_position"] = out_base
        return Z._z.inflate(C.byref(zs), Z.Z_NO_FLUSH)

    def next_():                                                 # GzipInputStream::Next: the bytes handed out, or None
        ok = st["zerror"] in (Z.Z_OK, Z.Z_STREAM_END, Z.Z_BUF_ERROR)
        if not ok or not zs.next_out:
            return None
        if zs.next_out != st["output_position"]:
            n = zs.next_out - st["output_position"]; b = C.string_at(st["output_position"], n); st["output_position"] = zs.next_out
            return b
        if st["zerror"] == Z.Z_STREAM_END:
            st["zerror"] = Z._z.inflateEnd(C.byref(zs))
            if st["zerror"] != Z.Z_OK:
                return None
            st["zerror"] = Z._init(zs, fmt)
            if st["zerror"] != Z.Z_OK:
                return None
        st["zerror"] = inflate_call()
        if st["zerror"] == Z.Z_STREAM_END and not zs.next_out:
            return None
        if st["zerror"] not in (Z.Z_OK, Z.Z_STREAM_END, Z.Z_BUF_ERROR):
            return None
        n = (zs.next_out or 0) - st["output_position"]; b = C.string_at(st["output_position"], n); st["output_position"] = zs.next_out
        return b

    try:
        while True:
            b = next_()
            if b is None:
                break
            got += b
        ok = fetched[0] == sum(len(b) for b in blocks) and next_() is None
    finally:
        if zs.state:
            Z._z.inflateEnd(C.byref(zs))
    return ok, bytes(got)


def oracle_echo_reply(conn, m, blob):
    """what an echo server with the gunzip step answers for one C oracle message m (offsets into blob) on oracle connection conn:
    the message inflated when the step inflates it, uncompressed (the echo sets no response_compress_type)"""
    (add, _, got), = server_step([m], blob, [False], 0, 1 << 30, 0)[0]   # (placement plays no part here)
    ok = (int(m["flags"]) & 3) == 3 and int(m["method_idx"]) >= 0 and (not int(m["flags"]) & 4 or add == F_GUNZIPPED)
    body = got if add == F_GUNZIPPED else bytes(blob[int(m["msg_off"]):int(m["msg_off"]) + int(m["msg_len"])])
    return conn.pack_response(int(m["stream_id"]), body if ok else b"", grpc_status=0 if ok else 12, grpc_message=b"" if ok else b"unimplemented")


class OracleGzEngine:
    """_h2loop.OracleEngine with the gunzip step: one C oracle H2Conn per TCP connection, echoes the inflated requests"""
    def __init__(self):
        self.conns = {}; self.n_compressed = 0

    def open(self, cid):
        self.conns[cid] = O.H2Conn()

    def feed(self, cid, buf):
        c = self.conns[cid]
        err, cons, msgs, ctrl, blob, _, _ = c.consume(buf)
        self.n_compressed += int(((msgs["flags"] & 4) != 0).sum())
        return cons, ctrl + b"".join(oracle_echo_reply(c, m, blob) for m in msgs), err, len(msgs)


class DeviceGzEngine:
    """_h2loop.DeviceEngine on connections opted in with h2_conn_set_gunzip: an inflated request is echoed from the device's out buffer
    (B2_H2_RESP_BODY_IN_OUT at its msg_off), a compressed one the device did not inflate is answered UNIMPLEMENTED like a failed call"""
    def __init__(self, ctx):
        import threading
        self.ctx = ctx
        self.lock = threading.Lock(); self.n_gunzipped = 0

    def open(self, cid):
        with self.lock:
            self.ctx.h2_conn_reset(cid); self.ctx.h2_conn_set_gunzip(cid)

    def feed(self, cid, buf):
        import numpy as np
        import brpc_b200
        from brpc_b200.abi import H2_RESPONSE_DT
        with self.lock:
            data, runs = brpc_b200.make_runs([buf]); runs["socket_id"] = cid
            rs, msgs, out = self.ctx.h2_process_batch(data, runs, msg_cap=1024, out_cap=8 << 20)
            ctrl = bytes(out[int(rs["ctrl_off"][0]):int(rs["ctrl_off"][0]) + int(rs["ctrl_len"][0])])
            reply = b""
            if len(msgs):
                ct = b"application/grpc"; gm = b"unimplemented"
                f = msgs["flags"]; gz = (f & F_GUNZIPPED) != 0
                self.n_gunzipped += int(gz.sum())
                r = np.zeros(len(msgs), H2_RESPONSE_DT)
                ok = ((f & 3) == 3) & (msgs["method_idx"] >= 0) & (((f & 4) == 0) | gz)
                r["conn"] = cid; r["stream_id"] = msgs["stream_id"]; r["status_code"] = 200
                r["flags"] = 1 | np.where(ok, np.where(((f & 16) != 0) & ~gz, 2, 4), 0)
                r["content_type_off"] = 0; r["content_type_len"] = len(ct)
                r["body_off"] = np.where(ok, msgs["msg_off"], 0); r["body_len"] = np.where(ok, msgs["msg_len"], 0)
                r["grpc_status"] = np.where(ok, 0, 12)
                r["grpc_message_off"] = len(ct); r["grpc_message_len"] = np.where(ok, 0, len(gm))
                reply = b"".join(self.ctx.h2_pack_responses(np.frombuffer(ct + gm + bytes(16), np.uint8), r))
            return int(rs["consumed"][0]), ctrl + reply, int(rs["parse_error"][0]), len(msgs)


def grpcio_gzip_client_calls(port, bodies, in_flight=128):
    """a grpcio channel with compression=Gzip: every body as one Echo call, up to `in_flight` at once; returns the replies in order"""
    import threading
    import grpc
    ch = grpc.insecure_channel("127.0.0.1:%d" % port, compression=grpc.Compression.Gzip,
                               options=[("grpc.max_receive_message_length", 1 << 24), ("grpc.max_send_message_length", 1 << 24)])
    try:
        call = ch.unary_unary("/example.EchoService/Echo", request_serializer=lambda b: b, response_deserializer=lambda b: b)
        gate = threading.BoundedSemaphore(in_flight); futs = []
        for b in bodies:
            gate.acquire()
            f = call.future(b, timeout=120)
            f.add_done_callback(lambda _f: gate.release())
            futs.append(f)
        return [f.result() for f in futs]
    finally:
        ch.close()


def echo_bodies(n, seed=5):
    """request bodies a gzip client compresses (text) and leaves alone (tiny, random): 0 B .. 60 KB"""
    import random
    rng = random.Random(seed)
    out = []
    for i in range(n):
        size = [0, 3, 100, 600, 4096, 20000, 60000][i % 7]
        out.append((b"message %d; " % i * (size // 12 + 1))[:size] if i % 3 else bytes(rng.randrange(256) for _ in range(size)))
    return out
