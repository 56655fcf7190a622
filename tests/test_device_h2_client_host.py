"""CPU: the DEVICE source of the client receive path (brpc_b200/csrc/b2_h2.cuh: k_h2_client_consume, k_h2_pack_req, k_h2_client_abandon)
built for the host — tests/cpp/gen_h2_host.py writes the harness, tests/cpp/h2_client_host.cc adds the client entry points — and checked two
ways that a GPU run cannot afford:
  * the recorded grpcio conversation (tests/golden/h2_client_rx_capture.json.gz) with every segment of the server's bytes cut at EVERY
    offset into two consecutive runs: each cut gives the same ctrl bytes, calls and leftover as the segment parsed whole, and the whole
    parse equals the oracle;
  * mutated server streams — frame lengths, types, flags and stream ids changed, bytes flipped, cut or repeated — against the oracle
    (tests/_h2client_oracle.py), call for call, with the device state memory pre-filled with a pattern."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
import _h2client_oracle as H  # noqa: E402
import _oracle as O  # noqa: E402
from _h2client_cases import mutate  # noqa: E402
from _h2client_loop import OracleClients, norm_device  # noqa: E402
from test_gpu_h2_client_rx import _capture, same  # noqa: E402
from brpc_b200.abi import H2_CALL_DT, H2_REQUEST_DT, H2_REQUEST_RESULT_DT, H2_RUN_STATUS_DT, RUN_DT  # noqa: E402

REGION = 1 << 21
CAP = 256


@pytest.fixture(scope="module")
def lib():
    cpp = os.path.join(HERE, "cpp")
    so = os.path.join(cpp, "libh2_client_host.so")
    deps = [os.path.join(cpp, f) for f in ("gen_h2_host.py", "h2_host_prelude.h", "h2_client_host.cc")] + \
           [os.path.join(ROOT, "brpc_b200", "csrc", f) for f in ("b2_h2.cuh", "b2_kernels.cuh", "b2_core.cuh", "b2_hpack_tables.cuh")] + \
           [os.path.join(ROOT, "include", "b2rpc.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([sys.executable, os.path.join(cpp, "gen_h2_host.py")])
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(cpp, "stub"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(cpp, "h2_client_host.cc")])
    l = C.CDLL(so)
    l.h2h_create.restype = C.c_void_p
    l.h2h_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint]
    l.h2h_destroy.argtypes = [C.c_void_p]
    l.h2c_client_reset.argtypes = [C.c_void_p, C.c_uint32]
    l.h2c_abandon.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    l.h2c_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.h2c_consume.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    l.h2c_snapshot.restype = C.c_void_p
    l.h2c_snapshot.argtypes = [C.c_void_p, C.c_uint32]
    l.h2c_restore.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    l.h2c_snap_free.argtypes = [C.c_void_p]
    l.h2c_every_offset.restype = C.c_uint32
    l.h2c_every_offset.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    return l


class HostClients:
    """DeviceClients of tests/_h2client_loop.py over the host-built kernels (pack returns status and stream id only)"""
    def __init__(self, lib, n, pending, stream_bytes, fill=0xa5):
        self.lib = lib
        self.h = lib.h2h_create(n, pending, stream_bytes, fill)
        for k in range(n):
            lib.h2c_client_reset(self.h, k)

    def pack(self, calls):
        blob, reqs = O.h2_request_blob(calls)
        reqs = reqs.astype(H2_REQUEST_DT); n = len(reqs)
        first = [i for i in range(n) if i == 0 or reqs[i]["conn"] != reqs[i - 1]["conn"]]
        g = np.array(first + [n], np.uint32)
        res = np.zeros(n, H2_REQUEST_RESULT_DT); off = 0
        for i in range(n):
            res[i]["out_off"] = off; off += (int(reqs[i]["body_len"]) * 2 + 8192 + 15) & ~15
        out = np.zeros(off + 16, np.uint8); data = np.frombuffer(blob, np.uint8)
        self.lib.h2c_pack(self.h, data.ctypes.data, reqs.ctypes.data, g.ctypes.data, len(first), out.ctypes.data, res.ctypes.data)
        # a "warp of one" runs lane 0, which does every state change of the request (stream id, windows, the pending stream, the HPACK
        # encoder); the frame bytes are written by the whole warp, so they are checked on the device and the emulated library, not here
        return [(int(r["status"]), int(r["stream_id"])) for r in res]

    def parse(self, chunks, region, call_cap):
        data = np.frombuffer(b"".join(chunks.values()) + bytes(64), np.uint8)
        runs = np.zeros(len(chunks), RUN_DT); off = 0
        for r, (k, b) in enumerate(chunks.items()):
            runs[r]["offset"] = off; runs[r]["length"] = len(b); runs[r]["socket_id"] = k; off += len(b)
        n = len(chunks)
        rs = np.zeros(n, H2_RUN_STATUS_DT); calls = np.zeros(call_cap * n, H2_CALL_DT); out = np.zeros(region * n, np.uint8)
        self.lib.h2c_consume(self.h, data.ctypes.data, runs.ctypes.data, n, rs.ctypes.data, calls.ctypes.data, call_cap, out.ctypes.data, region)
        res, got = [], []
        for r in range(n):
            s = rs[r]
            res.append((int(s["parse_error"]), int(s["consumed"]), out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()))
            got += [norm_device(c, out, data) for c in calls[r * call_cap:r * call_cap + int(s["n_msgs"])]]
        return res, got

    def abandon(self, conn, ids):
        ids = np.ascontiguousarray(ids, np.uint32)
        self.lib.h2c_abandon(self.h, conn, ids.ctypes.data, len(ids))

    def close(self):
        self.lib.h2h_destroy(self.h)


def _send(cl, k, step):
    return cl.pack([(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", b, e) for p, b, e in step[1]])


def test_capture_cut_at_every_offset_of_every_segment(lib):
    cap, steps = _capture()
    host = HostClients(lib, 1, cap["pending"], cap["stream_bytes"]); orc = OracleClients(1, cap["pending"], cap["stream_bytes"])
    rest = b""; total_cuts = 0; n_calls = 0
    for j, st in enumerate(steps):
        if st[0] == "send":
            assert _send(host, 0, st) == [x[:2] for x in _send(orc, 0, st)], j
            continue
        seg = st[1]
        bad, nc, left = C.c_uint32(), C.c_uint32(), C.c_uint32()
        snap = lib.h2c_snapshot(host.h, 0)
        n_bad = lib.h2c_every_offset(host.h, 0, rest, len(rest), seg, len(seg), 1, REGION, CAP, C.byref(bad), C.byref(nc), C.byref(left))
        assert n_bad == 0, (j, n_bad, bad.value, len(seg))
        assert nc.value == len(seg) + 1
        total_cuts += nc.value
        lib.h2c_restore(host.h, 0, snap); lib.h2c_snap_free(snap)
        dv, ov = host.parse({0: rest + seg}, REGION, CAP), orc.parse({0: rest + seg}, REGION, CAP)
        same(dv, ov, j)
        perr, cons, _ = dv[0][0]
        assert perr == H.NOT_ENOUGH_DATA and len(rest + seg) - cons == left.value
        rest = (rest + seg)[cons:]
        n_calls += len(dv[1])
    assert rest == b"" and total_cuts > 250000 and n_calls == sum(len(s[1]) for s in steps if s[0] == "send")
    host.close()


def test_mutated_server_streams_against_the_oracle(lib):
    cap, steps = _capture()
    recv_at = [j for j, s in enumerate(steps) if s[0] == "recv"]
    rng = random.Random(20261015)
    n_calls = 0; n_errors = 0
    for m in range(360):
        j = rng.choice(recv_at[:8] if m % 3 else recv_at)
        host = HostClients(lib, 2, cap["pending"], cap["stream_bytes"], fill=rng.choice([0x00, 0xa5, 0xff]))
        orc = OracleClients(2, cap["pending"], cap["stream_bytes"])
        rest = b""; ids = []
        for jj, st in enumerate(steps[:j + 3]):
            if st[0] == "send":
                d = _send(host, 1, st)
                assert d == [x[:2] for x in _send(orc, 1, st)], (m, jj)
                ids += [sid for _, sid in d]
                continue
            seg = mutate(rng, st[1], ids) if jj == j else st[1]
            chunks = {1: rest + seg}
            if jj == j and rng.random() < 0.3:                                   # and sometimes cut in two
                c = rng.randrange(len(chunks[1]) + 1)
                parts = [chunks[1][:c], chunks[1][c:]]
            else:
                parts = [chunks[1]]
            for pi, part in enumerate(parts):
                if pi:
                    part = rest + part
                dv, ov = host.parse({1: part}, REGION, CAP), orc.parse({1: part}, REGION, CAP)
                same(dv, ov, (m, jj, pi))
                perr, cons, _ = dv[0][0]
                n_calls += len(dv[1])
                if perr != H.NOT_ENOUGH_DATA:
                    n_errors += 1
                    rest = None
                    break
                rest = part[cons:]
            if rest is None:
                break
        host.close()
    assert n_calls > 3000 and n_errors > 20
