"""Test oracle for the receiving half of an h2 / gRPC client connection, written from the reference (apache/brpc) in plain Python:
ParseH2Message on a socket created by connect (src/brpc/policy/http2_rpc_protocol.cpp), OnEndStream / OnResetStream / OnGoAway, and what
ProcessHttpResponse (src/brpc/policy/http_rpc_protocol.cpp:349-564) decides before it parses the response body.  The request bytes come
from the C oracle's client side (_oracle.H2Conn.pack_request); HPACK decoding from the C oracle's decoder (_oracle.HPack).  The device's
capacities (stream pool, header record bytes, output space) are modelled so that runs that end in B2_PARSE_ERROR_NO_RESOURCE compare too."""
import _oracle as O

MAX_WINDOW = 0x7fffffff
HDR_BYTES = 4096                                  # B2_H2_HEADER_BYTES
ERR_MAX = 2048                                    # FLAGS_http_max_error_length
TRY_OTHERS, NOT_ENOUGH_DATA, NO_RESOURCE, ABSOLUTELY_WRONG = 1, 2, 4, 5   # B2_PARSE_ERROR_* (include/b2rpc.h)
ENDED, RESET_BY_PEER, RESET_BY_US, GOAWAY = 0, 1, 2, 3
F_GRPC, F_PREFIX_OK, F_COMPRESSED, F_BODY_IN_INPUT, F_HAS_GRPC_STATUS = 1, 2, 4, 16, 32
REQ_OK, REQ_ELIMIT, REQ_RUNOUT, REQ_LOGOFF, REQ_NO_ROOM = 0, 1, 2, 3, 4

# GrpcStatusToErrorCode (grpc.cpp:83-125): brpc errno values (errno.proto) and Linux ECANCELED / EINVAL / EEXIST / EPERM
GRPC_ERRNO = {0: 0, 1: 125, 3: 22, 4: 1008, 6: 17, 7: 1, 8: 2004, 12: 1002, 16: 1004}
GRPC_NAMES = ["OK", "CANCELED", "UNKNOWN", "INVALIDARGUMENT", "DEADLINEEXCEEDED", "NOTFOUND", "ALREADYEXISTS", "PERMISSIONDENIED",
              "RESOURCEEXHAUSTED", "FAILEDPRECONDITION", "ABORTED", "OUTOFRANGE", "UNIMPLEMENTED", "INTERNAL", "UNAVAILABLE", "DATALOSS",
              "UNAUTHENTICATED", "MAX"]                                          # GrpcStatusToString (grpc.cpp:29-51)
REASON = {100: "Continue", 101: "Switching Protocols", 200: "OK", 201: "Created", 202: "Accepted", 203: "Non-Authoritative Informational",
          204: "No Content", 205: "Reset Content", 206: "Partial Content", 300: "Multiple Choices", 301: "Move Permanently", 302: "Found",
          303: "See Other", 304: "Not Modified", 305: "Use Proxy", 307: "Temporary Redirect", 400: "Bad Request", 401: "Unauthorized",
          402: "Payment Required", 403: "Forbidden", 404: "Not Found", 405: "Method Not Allowed", 406: "Not Acceptable",
          407: "Proxy Authentication Required", 408: "Request Timeout", 409: "Conflict", 410: "Gone", 411: "Length Required",
          412: "Precondition Failed", 413: "Request Entity Too Large", 414: "Request-URI Too Long", 415: "Unsupported Media Type",
          416: "Requested Range Not Satisfiable", 417: "Expectation Failed", 500: "Internal Server Error", 501: "Not Implemented",
          502: "Bad Gateway", 503: "Service Unavailable", 504: "Gateway Timeout", 505: "HTTP Version Not Supported"}   # http_status_code.cpp
METHODS = [b"DELETE", b"GET", b"HEAD", b"POST", b"PUT", b"CONNECT", b"OPTIONS", b"TRACE", b"COPY", b"LOCK", b"MKCOL", b"MOVE", b"PROPFIND",
           b"PROPPATCH", b"SEARCH", b"UNLOCK", b"REPORT", b"MKACTIVITY", b"CHECKOUT", b"MERGE", b"M-SEARCH", b"NOTIFY", b"SUBSCRIBE",
           b"UNSUBSCRIBE", b"PATCH", b"PURGE", b"MKCALENDAR"]                     # Str2HttpMethod (http_method.cpp)


def cstr(b):
    k = b.find(b"\0")
    return b if k < 0 else b[:k]


def h2_status_of_error(e):                                                       # H2ErrorToStatusCode (http2.cpp:88-112)
    return {0: 200, 4: 504, 5: 400, 7: 503, 8: 503, 11: 503, 12: 401, 13: 505}.get(e, 500)


def strtol_int(v):
    """(int)strtol(c_str, NULL, 10)"""
    s = cstr(v); i = 0
    while i < len(s) and s[i] in b" \t\n\v\f\r":
        i += 1
    neg = False
    if i < len(s) and s[i] in b"+-":
        neg = s[i] == 45; i += 1
    j = i
    while j < len(s) and 48 <= s[j] <= 57:
        j += 1
    x = int(s[i:j]) if j > i else 0
    x = -x if neg else x
    x = max(-(1 << 63), min((1 << 63) - 1, x))
    x &= 0xffffffff
    return x - (1 << 32) if x & 0x80000000 else x


def header_ok(name, value):
    """one field of H2StreamContext::ConsumeHeaders (:1233-1282): False where it returns -1"""
    n = cstr(name)
    if not n or n[0] != 58:
        return True
    rest = n[1:]
    if rest in (b"authority", b"path", b"scheme"):
        return True
    if rest == b"method":
        return cstr(value).upper() in METHODS
    if rest == b"status":
        s = cstr(value); i = 0
        while i < len(s) and s[i] in b" \t\n\v\f\r":
            i += 1
        j = i + 1 if i < len(s) and s[i] in b"+-" else i
        d = j
        while d < len(s) and 48 <= s[d] <= 57:
            d += 1
        return (d if d > j else 0) == len(s)
    return False


def content_type_is_grpc(ct):
    """is_grpc_ct of ParseContentType (http_rpc_protocol.cpp:176-230): application/grpc, then the end, ';' or '+'"""
    ct = cstr(ct)
    return ct.startswith(b"application/grpc") and (len(ct) == 16 or ct[16:17] in (b";", b"+"))


def merge_headers(records):
    """HttpHeader as ConsumeHeaders fills it (:1233-1288, http_header.cpp:100-117).  Returns (merged records, status_code)."""
    status = 200
    out = []                                                                     # [name, value, kind]
    for name, value in records:
        n = cstr(name)
        if n[:1] == b":":
            if n == b":status":
                status = strtol_int(value)
            continue
        if n == b"content-type":                                                 # set_content_type: the last value wins
            for rec in out:
                if rec[2] == "ct":
                    rec[1] = value
                    break
            else:
                out.append([name, value, "ct"])
            continue
        if n.lower() == b"set-cookie":                                           # AddHeader: one each
            out.append([name, value, "sc"])
            continue
        for rec in out:                                                          # AppendHeader
            if rec[2] == "h" and cstr(rec[0]).lower() == n.lower():
                rec[1] = value if not rec[1] else rec[1] + (b"; " if n.lower() == b"cookie" else b",") + value
                break
        else:
            out.append([name, value, "h"])
    return [(a, b) for a, b, _ in out], status


def percent_decode(v):                                                           # PercentDecode (grpc.cpp:154-170)
    hx = lambda c: c - 87 if 97 <= c <= 102 else c - 55 if 65 <= c <= 70 else c - 48 if 48 <= c <= 57 else 0
    out = bytearray(); i = 0
    while i < len(v):
        c = v[i]
        if c == 37 and i + 2 < len(v):
            c = hx(v[i + 1]) * 16 + hx(v[i + 2]); i += 2
        out.append(c & 0xff); i += 1
    return bytes(out)


def get(merged, name):
    for n, v in merged:
        if cstr(n) == name:
            return v
    return None


def verdict(merged, sc, is_grpc, prefix_ok, compressed, msg, grpc_status):
    """ProcessHttpResponse (http_rpc_protocol.cpp:390-533) for a protobuf-typed call: (error code, text SetFailed gets)"""
    if is_grpc:
        if not prefix_ok:
            return 2002, b"Invalid gRPC response"
        if grpc_status is not None and grpc_status != 0:
            m = get(merged, b"grpc-message")
            text = cstr(percent_decode(m)) if m is not None else \
                ("GRPC_" + GRPC_NAMES[grpc_status] if 0 <= grpc_status < 18 else "Unknown-GrpcStatus").encode()
            return GRPC_ERRNO.get(grpc_status, 2001), text
    if sc < 200 or sc >= 300:
        rp = REASON.get(sc, "Unknown status code (%d)" % sc)
        err = b"HTTP/2.0 %d %s" % (sc, rp.encode())
        if msg:
            err += b": " + msg[:ERR_MAX]
        return 1010, cstr(err)
    if is_grpc and compressed and get(merged, b"grpc-encoding") is None:
        return 2002, b"Fail to find header `grpc-encoding' in compressed gRPC response"
    return 0, b""


def a16(n):
    return (n + 15) & ~15


class _Stream:
    def __init__(self, sid, window):
        self.sid = sid; self.records = []; self.hdr_len = 0; self.body = bytearray(); self.body_in = None
        self.ended = False; self.deferred = 0; self.window = window; self.abandoned = False


class ClientConn:
    """One client H2Context (H2Context(socket, NULL), :324-371) with the device's capacities."""

    def __init__(self, pending=8, stream_bytes=69632):
        self.tx = O.H2Conn(); self.hp = O.HPack(4096)
        self.P = pending; self.SB = stream_bytes
        self.streams = {}
        self.ready = False
        self.l_sws, self.l_mfs = 256 * 1024, 16384                             # _local_settings (H2Settings(), http2.cpp:26-34)
        self.r = dict(hts=4096, push=0, mcs=0xffffffff, sws=MAX_WINDOW, mfs=16384, mhl=0xffffffff)
        self.settings_received = False
        self.window = MAX_WINDOW                                                 # _remote_window_left
        self.deferred = 0                                                        # _deferred_window_update
        self.goaway = -1                                                         # _goaway_stream_id
        self.next_id = 1

    # ---- sending: H2UnsentRequest::AppendAndDestroySelf (:1496-1594) ----
    def pack_request(self, path, authority, body=b"", content_type=b"application/grpc", flags=1 | 8 | 16, extra=()):
        if len(self.streams) > self.r["mcs"]:                                   # (:1529-1531), no id consumed
            return REQ_ELIMIT, 0, b""
        if len(self.streams) >= self.P:                                          # device capacity
            return REQ_NO_ROOM, 0, b""
        data = len(body) + (5 if flags & 1 else 0)
        sid = self.next_id
        blocked = sid > 0x7fffffff or (data and (self.r["sws"] < data or self.window < data))
        if not blocked and self.goaway >= 0 and sid > self.goaway:
            self.tx.set_next_stream_id(sid + 2); self.next_id += 2
            if data:
                self.window -= data; self.tx.peer_update(conn_window_add=-data)
            return REQ_LOGOFF, sid, b""
        st, sid2, b = self.tx.pack_request(path, authority, body, content_type=content_type, flags=flags, extra=extra)
        if sid <= 0x7fffffff:
            self.next_id += 2
        if st != REQ_OK:
            return st, sid2, b
        assert sid2 == sid
        self.streams[sid] = _Stream(sid, self.r["sws"] - data)
        self.window -= data
        if self.deferred > 0:                                                    # ReleaseDeferredWindowUpdate in PackH2Message
            b += (4).to_bytes(3, "big") + b"\x08\x00" + (0).to_bytes(4, "big") + self.deferred.to_bytes(4, "big"); self.deferred = 0
        return st, sid, b

    def abandon(self, ids):                                                      # AddAbandonedStream (:1140-1143)
        for i in ids:
            if i in self.streams:
                self.streams[i].abandoned = True

    # ---- receiving ----
    def _wu(self, ctrl, sid, inc):
        ctrl += (4).to_bytes(3, "big") + b"\x08\x00" + sid.to_bytes(4, "big") + (inc & 0xffffffff).to_bytes(4, "big")

    def _defer(self, ctrl, size):                                                # DeferWindowUpdate (:1078-1095)
        if size <= 0:
            return
        self.deferred += size
        if self.deferred >= self.l_sws // 2:
            cw = self.deferred; self.deferred = 0
            if cw > 0:
                self._wu(ctrl, 0, cw)

    def _remove(self, ctrl, sid):                                                # RemoveStreamAndDeferWU (:373-386)
        s = self.streams.pop(sid, None)
        if s is not None:
            d = s.deferred; s.deferred = 0
            self._defer(ctrl, d)
        return s

    @staticmethod
    def _add_window(w, diff):                                                    # AddWindowSize (:261-281): (new value, ok)
        before = w; s = before + diff
        ok = True
        if ((before | diff) >> 31) & 1 == 0 and s & ~0x7fffffff:
            ok = False
        if ((before & diff) >> 31) & 1 == 1 and (s & ~0x7fffffff) == 0:
            ok = False
        return s, ok

    def _headers(self, s, frag):
        """ConsumeHeaders over one fragment into stream s: 0, -1 (error) or 'room' (device capacity)"""
        st, recs = self.hp.decode_block(frag)
        for name, value in recs:
            if s.hdr_len + 4 + len(name) + len(value) > HDR_BYTES:
                return "room"
            if not header_ok(name, value):
                return -1
            s.records.append((name, value)); s.hdr_len += 4 + len(name) + len(value)
        return -1 if st < 0 else 0

    def consume(self, data, run_off, run_len, r, region, call_cap):
        """One run of b2_h2_client_process_batch.  Returns (parse_error, consumed, calls, ctrl, blob bytes used)."""
        inp = bytes(data[run_off:run_off + run_len]); n = len(inp)
        ctrl = bytearray(); ctrl_cap = region // 4
        blob = [region // 4]; blob_end = region; gbase = r * region
        calls = []
        pos = last_ok = 0; perr = NOT_ENOUGH_DATA
        room = [False]

        def emit(s, how, status_override):
            in_input = s.body_in is not None
            need1 = a16(s.hdr_len) + (0 if in_input else a16(len(s.body)))
            if len(calls) >= call_cap or blob[0] + need1 > blob_end:
                return False
            merged, sc = merge_headers(s.records)
            if status_override is not None:
                sc = status_override
            body = bytes(data[s.body_in:s.body_in + s.body_len]) if in_input else bytes(s.body)
            ho = blob[0]; bo = ho + a16(s.hdr_len); eo = ho + need1
            c = dict(run_idx=r, stream_id=s.sid, how=how, status_code=sc, headers=merged, body=body, flags=F_BODY_IN_INPUT if in_input else 0,
                     headers_off=gbase + ho, body_off=s.body_in if in_input else gbase + bo, msg=b"", msg_off=0)
            ct = get(merged, b"content-type")
            is_grpc = ct is not None and content_type_is_grpc(ct)
            prefix_ok = compressed = False; msg = body
            if is_grpc:
                c["flags"] |= F_GRPC
                if not body:
                    prefix_ok = True; c["msg_off"] = c["body_off"]
                elif len(body) >= 5:
                    compressed = body[0] != 0
                    if int.from_bytes(body[1:5], "big") + 5 == len(body):
                        prefix_ok = True; c["msg_off"] = c["body_off"] + 5; c["msg"] = body[5:]
                if prefix_ok:
                    c["flags"] |= F_PREFIX_OK; msg = c["msg"]
                if compressed:
                    c["flags"] |= F_COMPRESSED
            gs = get(merged, b"grpc-status")
            c["grpc_status"] = strtol_int(gs) if gs is not None else -1
            if gs is not None:
                c["flags"] |= F_HAS_GRPC_STATUS
            code, text = verdict(merged, sc, is_grpc, prefix_ok, compressed, msg, c["grpc_status"] if gs is not None else None)
            if eo + a16(len(text)) > blob_end:
                return False
            c["error_code"] = code; c["error"] = text; c["error_off"] = gbase + eo if text else 0
            blob[0] = eo + a16(len(text))
            calls.append(c)
            return True

        def ack(b):
            if len(ctrl) + len(b) > ctrl_cap:
                room[0] = True
                return
            ctrl.extend(b)

        def clear_abandoned():                                                   # ClearAbandonedStreams (:1145-1157)
            for sid in sorted(k for k, s in self.streams.items() if s.abandoned):
                rctl = bytearray(); self._remove(rctl, sid); ack(bytes(rctl))
        n_cleared = 0
        while True:
            if len(calls) != n_cleared:                                          # ParseH2Message returned a message: it clears
                clear_abandoned(); n_cleared = len(calls)
            if room[0]:
                perr = NO_RESOURCE; break
            if not self.ready:
                self.ready = True; last_ok = pos; continue
            left = n - pos
            if left < 3:
                break
            length = int.from_bytes(inp[pos:pos + 3], "big")
            if length > self.l_mfs:
                perr = ABSOLUTELY_WRONG; break
            if left - 3 < 6 + length:
                break
            ftype, flags, sid = inp[pos + 3], inp[pos + 4], int.from_bytes(inp[pos + 5:pos + 9], "big")
            if sid & 0x80000000:
                perr = ABSOLUTELY_WRONG; break
            pos += 9
            if ftype > 9:
                perr = ABSOLUTELY_WRONG; break
            pl = inp[pos:pos + length]
            used = 0
            err = None; done = None                                              # err: (h2 error, stream id or 0); done: (stream, how, status)
            goaway = None
            out = bytearray()
            if ftype == 0:                                                       # OnData (:699-779)
                frag = length; padl = 0
                if flags & 8 and length == 0:
                    err = (6, 0)
                else:
                    if flags & 8:
                        frag -= 1; padl = pl[0]; used = 1
                    if frag < padl:
                        err = (6, 0)
                    else:
                        frag -= padl
                        s = self.streams.get(sid)
                        if s is None:
                            used += frag + padl
                            quota = self.l_sws // (len(self.streams) + 1)
                            tmp = frag
                            if frag >= quota:
                                if frag > self.l_sws:
                                    self._defer(out, tmp); err = (5, sid)
                                else:
                                    swu = tmp; tmp = 0
                                    if swu > 0:
                                        self._wu(out, sid, swu); cw = swu + self.deferred; self.deferred = 0; self._wu(out, 0, cw)
                            if err is None:
                                self._defer(out, tmp); err = (5, sid)
                        else:
                            if not s.body and s.body_in is None and flags & 1 and frag:
                                s.body_in = run_off + pos + used; s.body_len = frag
                            elif HDR_BYTES + len(s.body) + frag > self.SB:
                                room[0] = True
                            else:
                                s.body += pl[used:used + frag]
                            if not room[0]:
                                used += frag + padl
                                acc = frag + s.deferred; s.deferred += frag
                                quota = self.l_sws // (len(self.streams) + 1)
                                if acc >= quota and acc > self.l_sws:
                                    err = (3, sid)
                                else:
                                    if acc >= quota:
                                        swu = s.deferred; s.deferred = 0
                                        if swu > 0:
                                            self._wu(out, sid, swu); cw = swu + self.deferred; self.deferred = 0; self._wu(out, 0, cw)
                                    if flags & 1:
                                        s2 = self._remove(out, sid)
                                        if s2 is not None:
                                            done = (s2, ENDED, None)
            elif ftype == 1:                                                     # OnHeaders (:545-653), client side
                if sid == 0:
                    err = (1, 0)
                else:
                    pad, pri = flags & 8, flags & 0x20
                    if length < (5 if pri else 0) + (1 if pad else 0):
                        err = (6, 0)
                    else:
                        frag = length; padl = 0
                        if pad:
                            padl = pl[0]; used = 1; frag -= 1
                        if pri:
                            used += 5; frag -= 5
                        if frag < padl:
                            err = (6, 0)
                        else:
                            frag -= padl
                            s = self.streams.get(sid)
                            if s is None:                                        # decoded and dropped (:600-606)
                                if blob[0] + HDR_BYTES > blob_end:
                                    room[0] = True
                                else:
                                    rc = self._headers(_Stream(sid, 0), pl[used:used + frag])
                                    if rc == "room":
                                        room[0] = True
                                    elif rc == 0:
                                        used += frag + padl
                            else:
                                rc = self._headers(s, pl[used:used + frag])
                                if rc == "room":
                                    room[0] = True
                                elif rc < 0:
                                    err = (1, 0)
                                else:
                                    used += frag + padl
                                    if flags & 4:
                                        if flags & 1:
                                            s2 = self._remove(out, sid)
                                            if s2 is not None:
                                                done = (s2, ENDED, None)
                                    elif flags & 1:
                                        s.ended = True
            elif ftype in (2, 5):                                                # OnPriority / OnPushPromise
                err = (1, 0)
            elif ftype == 3:                                                     # OnResetStream (:781-823)
                if length != 4:
                    err = (6, 0)
                else:
                    used = 4
                    s2 = self._remove(out, sid)
                    if s2 is not None:
                        done = (s2, RESET_BY_PEER, h2_status_of_error(int.from_bytes(pl[:4], "big")))
            elif ftype == 4:                                                     # OnSettings (:848-916)
                if sid != 0:
                    err = (1, 0)
                elif flags & 1:
                    if length != 0:
                        err = (1, 0)
                    else:
                        self.l_sws, self.l_mfs = 256 * 1024, 16384               # _local_settings = _unack_local_settings
                else:
                    old = self.r["sws"]
                    t = dict(hts=4096, push=0, mcs=0xffffffff, sws=256 * 1024, mfs=16384, mhl=0xffffffff) if not self.settings_received else dict(self.r)
                    ok = length % 6 == 0
                    if ok:
                        for i in range(length // 6):
                            ident = int.from_bytes(pl[used:used + 2], "big"); v = int.from_bytes(pl[used + 2:used + 6], "big"); used += 6
                            if ident == 1:
                                t["hts"] = v
                            elif ident == 2:
                                if v > 1:
                                    ok = False; break
                                t["push"] = v
                            elif ident == 3:
                                t["mcs"] = v
                            elif ident == 4:
                                if v > MAX_WINDOW:
                                    ok = False; break
                                t["sws"] = v
                            elif ident == 5:
                                if v > 16777215 or v < 16384:
                                    ok = False; break
                                t["mfs"] = v
                            elif ident == 6:
                                t["mhl"] = v
                    first = not self.settings_received
                    if first and not ok:
                        err = (1, 0)
                    else:
                        if first:
                            self.window -= MAX_WINDOW - 65535; self.settings_received = True
                            self.tx.peer_update(conn_window_add=-(MAX_WINDOW - 65535))
                        self.r = t
                        self.tx.peer_update(header_table_size=t["hts"], max_frame_size=t["mfs"], stream_window_size=t["sws"])
                        if not ok:
                            err = (1, 0)
                        else:
                            diff = self.r["sws"] - old
                            flow_ok = True
                            if diff:
                                for s in self._slot_order():
                                    s.window, good = self._add_window(s.window, diff)
                                    if not good:
                                        flow_ok = False; break
                            if not flow_ok:
                                err = (3, 0)
                            else:
                                out += b"\0\0\0\x04\x01\0\0\0\0"
            elif ftype == 6:                                                     # OnPing (:930-952)
                if length != 8:
                    err = (6, 0)
                elif sid != 0:
                    err = (1, 0)
                elif not flags & 1:
                    out += b"\0\0\x08\x06\x01\0\0\0\0" + pl[:8]; used = 8
            elif ftype == 7:                                                     # OnGoAway (:959-1006), client side
                if length < 8:
                    err = (6, 0)
                elif sid != 0 or flags:
                    err = (1, 0)
                else:
                    used = length
                    last = int.from_bytes(pl[length - 8:length - 4], "big")
                    goaway = last - (1 << 32) if last & 0x80000000 else last
            elif ftype == 8:                                                     # OnWindowUpdate (:1008-1038)
                if length != 4:
                    err = (6, 0)
                else:
                    inc = int.from_bytes(pl[:4], "big"); used = 4
                    if inc & 0x80000000 or inc == 0:
                        err = (1, 0)
                    elif sid == 0:
                        self.window, good = self._add_window(self.window, inc)
                        self.tx.peer_update(conn_window_add=inc)
                        if not good:
                            err = (3, 0)
                    elif sid in self.streams:
                        s = self.streams[sid]
                        s.window, good = self._add_window(s.window, inc)
                        if not good:
                            err = (3, 0)
            elif ftype == 9:                                                     # OnContinuation (:655-697)
                used = length
                s = self.streams.get(sid)
                if s is None:
                    if blob[0] + HDR_BYTES > blob_end:
                        room[0] = True
                    elif self._headers(_Stream(sid, 0), pl) == "room":
                        room[0] = True
                else:
                    rc = self._headers(s, pl)
                    if rc == "room":
                        room[0] = True
                    elif rc < 0:
                        err = (1, 0)
                    elif flags & 4 and s.ended:
                        s2 = self._remove(out, sid)
                        if s2 is not None:
                            done = (s2, ENDED, None)
            ack(bytes(out))
            if room[0]:
                continue
            pos += used
            if err is not None:
                e, esid = err
                if esid:
                    ack((4).to_bytes(3, "big") + b"\x03\x00" + esid.to_bytes(4, "big") + e.to_bytes(4, "big"))
                    rctl = bytearray(); s2 = self._remove(rctl, esid); ack(bytes(rctl))
                    last_ok = pos
                    if s2 is not None and not emit(s2, RESET_BY_US, h2_status_of_error(e)):
                        room[0] = True
                else:
                    ack((8).to_bytes(3, "big") + b"\x07\x00" + b"\0\0\0\0" + b"\xff\xff\xff\xff" + e.to_bytes(4, "big"))
                    last_ok = pos
                continue
            last_ok = pos
            if goaway is not None:                                               # SetLogOff + RemoveGoAwayStreams (:388-414)
                self.goaway = goaway
                for gsid in sorted(k for k in self.streams if k > goaway):
                    s2 = self.streams.pop(gsid)
                    if not emit(s2, GOAWAY, 503):
                        room[0] = True; break
                continue
            if done is not None and not emit(*done):
                room[0] = True
        clear_abandoned()
        if room[0]:
            perr = NO_RESOURCE
        return perr, last_ok, calls, bytes(ctrl), blob[0] - region // 4

    def _slot_order(self):
        return list(self.streams.values())
