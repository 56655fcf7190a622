"""Hand-built server frames for the receiving half of an h2 client connection: what a well-behaved server does not send (resets, GOAWAY,
headers on unknown streams, bad :status, broken gRPC prefixes, error statuses with long bodies, settings / pings / window updates,
abandoned streams).  Each case takes a client (oracle or device adapter of tests/_h2client_loop.py) and a connection index, opens
calls on it and returns the server's bytes as the chunks to parse, in order."""
from _h2client_loop import ECHO, GRPC_EXTRA

STREAM_BYTES = (512 << 10) + 4096          # the pool the cases are written for: 8 pending streams of up to 512 KiB


def frame(t, flags, sid, payload):
    return len(payload).to_bytes(3, "big") + bytes([t, flags]) + sid.to_bytes(4, "big") + payload


def lit(name, value):                                                            # literal without indexing, new name, no Huffman
    return b"\x00" + bytes([len(name)]) + name + bytes([len(value)]) + value


def lit_inc(name, value):                                                        # literal with incremental indexing, new name
    return b"\x40" + bytes([len(name)]) + name + bytes([len(value)]) + value


def grpc_body(msg, flag=0):
    return bytes([flag]) + len(msg).to_bytes(4, "big") + msg


OK_HDRS = b"\x88" + lit(b"content-type", b"application/grpc")                    # :status 200 (static 8)


def trailers(status=b"0", message=None):
    return lit(b"grpc-status", status) + (lit(b"grpc-message", message) if message is not None else b"")


def new_conn(cl, k, n_calls=4):
    res = cl.pack([(k, 1 | 8 | 16, ECHO, b"h:1", b"application/grpc", b"q", GRPC_EXTRA) for _ in range(n_calls)])
    assert all(st == 0 for st, _, _ in res)
    return [sid for _, sid, _ in res]


HAND_CASES = []


def hand(f):
    HAND_CASES.append(f)
    return f


@hand
def case_unary_ok_and_trailers_merge(cl, k):
    ids = new_conn(cl, k)
    hdr = OK_HDRS + lit(b"x-dup", b"a") + lit(b"cookie", b"k=1") + lit(b"set-cookie", b"s=1") + lit(b"x-empty", b"")
    tr = trailers() + lit(b"x-dup", b"b") + lit(b"cookie", b"k=2") + lit(b"set-cookie", b"s=2") + lit(b"x-empty", b"z") + \
        lit(b"content-type", b"application/grpc+proto")
    data = frame(1, 4, ids[0], hdr) + frame(0, 0, ids[0], grpc_body(b"hello")) + frame(1, 5, ids[0], tr)
    return [data]


@hand
def case_rst_stream_from_peer_and_unknown(cl, k):
    ids = new_conn(cl, k)
    data = frame(1, 4, ids[0], OK_HDRS) + frame(3, 0, ids[0], (8).to_bytes(4, "big")) + frame(3, 0, 99, (2).to_bytes(4, "big")) + \
        frame(3, 0, ids[1], (7).to_bytes(4, "big")) + frame(3, 0, ids[2], b"\0\0\0")
    return [data]


@hand
def case_goaway_above_and_below(cl, k):
    ids = new_conn(cl, k, 6)
    data = frame(1, 5, ids[0], OK_HDRS + trailers()) + frame(7, 0, 0, b"debug data" + ids[2].to_bytes(4, "big") + (0).to_bytes(4, "big")) + \
        frame(1, 5, ids[1], OK_HDRS + trailers(b"5"))
    return [data]


@hand
def case_goaway_last_stream_id_with_the_high_bit(cl, k):
    """last_stream_id is read as an int (:975): 0x80000000 .. 0xfffffffe are negative, so every pending stream leaves and no later
    request is refused (TryToInsertStream checks _goaway_stream_id >= 0); free stream records must not be taken for streams"""
    ids = new_conn(cl, k, 2)
    return [frame(7, 0, 0, (0xfffffffe).to_bytes(4, "big") + (2).to_bytes(4, "big")),
            frame(7, 0, 0, b"dbg" + (0x80000000).to_bytes(4, "big") + (0).to_bytes(4, "big")) + frame(1, 5, ids[0], OK_HDRS + trailers())]


@hand
def case_goaway_zero_takes_all(cl, k):
    ids = new_conn(cl, k, 5)
    return [frame(1, 4, ids[3], OK_HDRS) + frame(0, 0, ids[3], grpc_body(b"partial")) + frame(7, 0, 0, bytes(8))]


@hand
def case_headers_on_unknown_streams_advance_hpack(cl, k):
    ids = new_conn(cl, k)
    data = frame(1, 4, 77, lit_inc(b"x-table", b"v1")) + frame(1, 0, 79, lit_inc(b"x-more", b"v2")) + frame(9, 4, 79, lit_inc(b"x-cont", b"v3")) + \
        frame(1, 5, ids[0], OK_HDRS + b"\xbe\xbf\xc0" + trailers())              # the three entries by index (62, 63, 64)
    return [data]


@hand
def case_bad_status_and_unknown_pseudo(cl, k):
    ids = new_conn(cl, k)
    data = frame(1, 5, ids[0], lit(b":status", b"20x")) + frame(1, 5, ids[1], lit(b":status", b" +204")) + \
        frame(1, 5, ids[2], lit(b":bogus", b"1")) + frame(1, 5, ids[3], lit(b":status", b"99999999999999"))
    return [data]


@hand
def case_grpc_prefix_missing_short_and_compressed(cl, k):
    ids = new_conn(cl, k)
    data = frame(1, 4, ids[0], OK_HDRS) + frame(0, 1, ids[0], b"abc") + \
        frame(1, 4, ids[1], OK_HDRS) + frame(0, 1, ids[1], grpc_body(b"12345")[:-1]) + \
        frame(1, 4, ids[2], OK_HDRS) + frame(0, 0, ids[2], grpc_body(b"zz", 1)) + frame(1, 5, ids[2], trailers()) + \
        frame(1, 4, ids[3], OK_HDRS + lit(b"grpc-encoding", b"gzip")) + frame(0, 0, ids[3], grpc_body(b"zz", 1)) + frame(1, 5, ids[3], trailers())
    return [data]


@hand
def case_non_2xx_with_long_body_and_percent_message(cl, k):
    ids = new_conn(cl, k)
    long_body = bytes(65 + i % 26 for i in range(3000))
    data = frame(1, 4, ids[0], b"\x8d" + lit(b"content-type", b"text/plain")) + frame(0, 1, ids[0], long_body) + \
        frame(1, 5, ids[1], lit(b":status", b"418")) + \
        frame(1, 5, ids[2], OK_HDRS + trailers(b"14", b"down%20for%2Gmaint%e2%9c%93%")) + \
        frame(1, 5, ids[3], OK_HDRS + trailers(b"3"))
    return [data]


@hand
def case_settings_ack_ping_window_update(cl, k):
    ids = new_conn(cl, k)
    data = frame(4, 0, 0, (3).to_bytes(2, "big") + (2).to_bytes(4, "big") + (4).to_bytes(2, "big") + (1 << 20).to_bytes(4, "big") +
                 (5).to_bytes(2, "big") + (32768).to_bytes(4, "big")) + frame(4, 1, 0, b"") + frame(6, 0, 0, b"12345678") + \
        frame(8, 0, 0, (1000).to_bytes(4, "big")) + frame(8, 0, ids[0], (5).to_bytes(4, "big")) + \
        frame(4, 1, 0, b"x") + frame(2, 0, ids[1], bytes(5)) + frame(6, 1, 0, b"ackackac")     # (an ack's payload stays unread: last)
    return [data]


@hand
def case_data_on_unknown_stream_and_window_updates(cl, k):
    ids = new_conn(cl, k)
    data = frame(0, 0, 1001, b"x" * 100) + frame(1, 4, ids[0], OK_HDRS)
    big = frame(0, 0, ids[0], b"y" * 16384) * 17                                 # more than the 256 KiB local stream window in all
    return [data, big]


@hand
def case_abandoned_streams(cl, k):
    ids = new_conn(cl, k)
    cl.abandon(k, [ids[1], ids[2], 12345])
    data = frame(1, 4, ids[1], OK_HDRS) + frame(0, 0, ids[1], b"z" * 16000) + frame(1, 5, ids[0], OK_HDRS + trailers())
    return [data, frame(1, 5, ids[1], OK_HDRS + trailers())]


@hand
def case_abandoned_stream_completing_first_is_reported(cl, k):
    """ParseH2Message clears abandoned streams each time it returns a message: an abandoned call that completes first is still
    reported, one that completes after another call of the same run is gone"""
    ids = new_conn(cl, k)
    cl.abandon(k, [ids[0], ids[2]])
    return [frame(1, 5, ids[0], OK_HDRS + trailers()) + frame(1, 5, ids[1], OK_HDRS + trailers()) + frame(1, 5, ids[2], OK_HDRS + trailers())]




# ---- mutations of recorded server streams -------------------------------------------------------------------------------------------
def _frames(seg):
    """offsets of the frame heads at the front of seg"""
    out = []; p = 0
    while len(seg) - p >= 9:
        n = int.from_bytes(seg[p:p + 3], "big")
        out.append(p)
        if len(seg) - p < 9 + n:
            break
        p += 9 + n
    return out


def mutate(rng, seg, ids):
    """seg with one change a faulty or hostile server could make: a frame head field, a payload byte, a cut, a repeated frame, or a
    hand-made frame (GOAWAY with the high bit set in last_stream_id, RST_STREAM, SETTINGS ACK, PING) put in between"""
    b = bytearray(seg)
    heads = _frames(seg) or [0]
    h = rng.choice(heads)
    kind = rng.randrange(9)
    if kind == 0 and len(b) >= h + 3:                                            # frame length
        n = int.from_bytes(b[h:h + 3], "big")
        n = rng.choice([0, 1, 4, 5, 7, 8, 9, n - 1, n + 1, n + 9, 16384, 16385, rng.randrange(1 << 24)]) & 0xffffff
        b[h:h + 3] = max(0, n).to_bytes(3, "big")
    elif kind == 1 and len(b) > h + 3:                                           # frame type
        b[h + 3] = rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 255])
    elif kind == 2 and len(b) > h + 4:                                           # flags
        b[h + 4] = rng.choice([0, 1, 4, 5, 8, 0x20, 0x25, 0x2d, 255])
    elif kind == 3 and len(b) >= h + 9:                                          # stream id
        sid = rng.choice([0, 1, 2, 99, 0x7fffffff, 0x80000000, 0xfffffffe, 0xffffffff] + ids)
        b[h + 5:h + 9] = sid.to_bytes(4, "big")
    elif kind == 4 and b:                                                        # a bit anywhere
        i = rng.randrange(len(b)); b[i] ^= 1 << rng.randrange(8)
    elif kind == 5 and b:                                                        # a byte of a payload's first bytes (HPACK, settings, goaway)
        i = min(len(b) - 1, h + 9 + rng.randrange(12)); b[i] = rng.randrange(256)
    elif kind == 6:                                                              # cut
        del b[rng.randrange(len(b) + 1):]
    elif kind == 7 and len(heads) > 1:                                           # a frame twice
        k = heads.index(h); e = heads[k + 1] if k + 1 < len(heads) else len(b)
        b[e:e] = b[h:e]
    else:                                                                        # a hand-made frame in between
        f = rng.choice([bytes.fromhex("000008070000000000") + rng.choice([b"\x80\0\0\0", b"\xff\xff\xff\xfe", b"\0\0\0\x03"]) + b"\0\0\0\0",
                        bytes.fromhex("000004030000000001") + b"\0\0\0\x08", bytes.fromhex("000000040100000000"),
                        bytes.fromhex("0000080600000000001122334455667788")])
        b[h:h] = f
    return bytes(b)
