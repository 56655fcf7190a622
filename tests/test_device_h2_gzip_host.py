"""CPU: the DEVICE source of the gunzip passes (brpc_b200/csrc/b2_h2.cuh: k_h2_gz_select, k_h2_gz_size, k_h2_gz_place, k_h2_gz_inflate)
built for the host — tests/cpp/gen_h2_host.py writes the harness, tests/cpp/h2_gzip_host.cc launches the passes after k_h2_client_consume as
b2_api.cu does — against the oracle (tests/_h2gzip.py), call for call with msg_off and the inflated bytes: the cases of
tests/test_gpu_h2_gzip.py plus a larger mutation corpus (bit flips, byte changes and cuts of streams of every block type), with the device
state memory pre-filled with a pattern."""
import ctypes as C
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
import _h2gzip as G  # noqa: E402
from _h2client_cases import grpc_body, trailers  # noqa: E402
from test_device_h2_client_host import HostClients  # noqa: E402
from test_gpu_h2_gzip import GZ_HDRS, GzOracle, client_cases, client_replies, gz, norm, same  # noqa: E402
from brpc_b200.abi import H2_CALL_DT, H2_RUN_STATUS_DT, RUN_DT  # noqa: E402

REGION = 1 << 20
CAP = 64
PENDING, STREAM_BYTES = 64, (256 << 10) + 4096


@pytest.fixture(scope="module")
def lib():
    cpp = os.path.join(HERE, "cpp")
    so = os.path.join(cpp, "libh2_gzip_host.so")
    deps = [os.path.join(cpp, f) for f in ("gen_h2_host.py", "h2_host_prelude.h", "h2_client_host.cc", "h2_gzip_host.cc")] + \
           [os.path.join(ROOT, "brpc_b200", "csrc", f) for f in ("b2_h2.cuh", "b2_kernels.cuh", "b2_core.cuh", "b2_hpack_tables.cuh", "b2_inflate.cuh")] + \
           [os.path.join(ROOT, "include", "b2rpc.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([sys.executable, os.path.join(cpp, "gen_h2_host.py")])
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(cpp, "stub"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(cpp, "h2_gzip_host.cc")])
    l = C.CDLL(so)
    l.h2h_create.restype = C.c_void_p
    l.h2h_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint]
    l.h2h_destroy.argtypes = [C.c_void_p]
    l.h2c_client_reset.argtypes = [C.c_void_p, C.c_uint32]
    l.h2c_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.h2g_set_gunzip.argtypes = [C.c_void_p, C.c_uint32, C.c_int]
    l.h2g_consume.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                              C.c_void_p, C.c_void_p]
    return l


class HostGz(HostClients):
    """the host-built kernels with gunzip on the given connections; parse compacts nothing (per-run slots, like the kernels see them)"""
    def __init__(self, lib, n, on, fill=0xa5):
        super().__init__(lib, n, PENDING, STREAM_BYTES, fill)
        for k in on:
            lib.h2g_set_gunzip(self.h, k, 1)

    def pack(self, calls):
        return [(st, sid, b"") for st, sid in super().pack(calls)]

    def parse(self, chunks, region, call_cap):
        data = np.frombuffer(b"".join(chunks.values()) + bytes(64), np.uint8)
        runs = np.zeros(len(chunks), RUN_DT); off = 0
        for r, (k, b) in enumerate(chunks.items()):
            runs[r]["offset"] = off; runs[r]["length"] = len(b); runs[r]["socket_id"] = k; off += len(b)
        n = len(chunks)
        rs = np.zeros(n, H2_RUN_STATUS_DT); calls = np.zeros(call_cap * n, H2_CALL_DT); out = np.full(region * n, 0x5a, np.uint8)
        scratch = np.full(n * 4096, 0xa5, np.uint8); gzw = np.full(call_cap * n, 0xa5a5a5a5, np.uint32)
        self.lib.h2g_consume(self.h, data.ctypes.data, runs.ctypes.data, n, rs.ctypes.data, calls.ctypes.data, call_cap, out.ctypes.data, region,
                             scratch.ctypes.data, gzw.ctypes.data)
        res, got = [], []
        for r in range(n):
            s = rs[r]
            res.append((int(s["parse_error"]), int(s["consumed"]), out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()))
            got += [norm(c, out, data) for c in calls[r * call_cap:r * call_cap + int(s["n_msgs"])]]
        return res, got


def mutated_corpus(rng, n):
    """(compressed stream) mutations of streams of every block type: bit flips, byte changes, cuts, duplicated and dropped ranges"""
    seeds = [gz(p, level=lv, strategy=st) for p in (b"mutation corpus text " * 60, bytes(rng.randrange(256) for _ in range(900)), b"\7" * 5000)
             for lv, st in ((6, zlib.Z_DEFAULT_STRATEGY), (0, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED))]
    out = []
    for i in range(n):
        b = bytearray(rng.choice(seeds)); k = rng.random()
        if k < 0.4:
            for _ in range(rng.randrange(1, 4)):
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        elif k < 0.6:
            b[rng.randrange(len(b))] = rng.randrange(256)
        elif k < 0.8:
            b = b[:rng.randrange(len(b))]
        else:
            a = rng.randrange(len(b)); z = rng.randrange(a, min(len(b), a + 40) + 1)
            b = b[:a] + b[z:] if rng.random() < 0.5 else b[:z] + b[a:]
        out.append(bytes(b))
    return out


def _compare(lib, cases, region=REGION):
    n = len(cases); on = set(range(0, n, 2)) | {n - 1}
    host = HostGz(lib, n, on); orc = GzOracle(n, on, PENDING, STREAM_BYTES)
    chunks = {k: client_replies(host, k, cases[k]) for k in range(n)}
    assert chunks.keys() == {k: client_replies(orc, k, cases[k]) for k in range(n)}.keys()
    hv, ov = host.parse(chunks, region, CAP), orc.parse(chunks, region, CAP)
    host.close()
    same(hv, ov, "host")
    return [c for c in hv[1] if c["run_idx"] in on]


def test_gpu_file_cases_on_the_host_build(lib):
    got = _compare(lib, client_cases(random.Random(20261015)))
    assert sum(1 for c in got if c["flags"] & G.F_GUNZIPPED) > 20


def test_mutation_corpus_on_the_host_build(lib):
    rng = random.Random(4)
    corpus = mutated_corpus(rng, 600)
    cases = [[(GZ_HDRS, grpc_body(s, 1), trailers()) for s in corpus[at:at + 40]] for at in range(0, len(corpus), 40)]
    got = _compare(lib, cases)
    n_short = sum(1 for c in got if c["flags"] & G.F_GUNZIPPED and len(c["msg"]) < 900)
    assert sum(1 for c in got if c["flags"] & G.F_GUNZIPPED) > 250 and n_short > 50
