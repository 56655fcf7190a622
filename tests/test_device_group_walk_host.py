"""CPU: the group walk of k_tile_walk (one thread walks the frame chain across G consecutive tiles of a connection from the speculative
entry of the group's first tile, DESIGN §3) from a host-compilable copy of brpc_b200/csrc/b2_kernels.cuh (tests/cpp/gen_kernels_host.py),
then k_resolve and k_frame_table.  The group heads' entries are hostile — true frame starts, random positions, frame look-alikes in
payloads, later frame starts, none — on five-protocol traffic with garbage and truncation, client runs included: the runs and the frame
table must be the oracle's every time, and every member the walk entered must hold what the per-tile walk writes from the same entry."""
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
import _oracle as O  # noqa: E402
from _traffic import SEED, echo_frame, mixed_frames, rnd62  # noqa: E402
from brpc_b200.abi import RUN_STATUS_DT  # noqa: E402
from brpc_b200.messenger import make_runs  # noqa: E402
from test_core_cut_host import ALL, five_protocol_stream  # noqa: E402

NONE = 0xffffffff


@pytest.fixture(scope="module")
def gw():
    cpp = os.path.join(HERE, "cpp")
    so = os.path.join(cpp, "libgroup_walk_host.so")
    deps = [os.path.join(cpp, f) for f in ("gen_kernels_host.py", "kernels_host_prelude.h", "h2_host_prelude.h", "group_walk_host.cc")] + \
           [os.path.join(ROOT, "brpc_b200", "csrc", f) for f in ("b2_kernels.cuh", "b2_core.cuh", "b2_inflate.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([sys.executable, os.path.join(cpp, "gen_kernels_host.py")])
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(cpp, "stub"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(cpp, "group_walk_host.cc")])
    lib = C.CDLL(so)
    lib.kh_front_group.restype = C.c_int
    lib.kh_front_group.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    lib.kh_group_vs_tiles.restype = C.c_int
    lib.kh_group_vs_tiles.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32,
                                      C.c_void_p, C.POINTER(C.c_uint32)]
    return lib


def traffic(rng, kind):
    """(streams, protocol mask, client runs?): the four kinds of the per-tile exactness test, and client runs with all five handlers."""
    fake = echo_frame(rng, 5, b"x" * 30)
    if kind == 0: streams = [b"".join(mixed_frames(rng, rng.randrange(5, 80), big=rng.random() < 0.3)) for _ in range(8)]
    elif kind in (1, 4): streams = [b"".join(five_protocol_stream(rng, rng.randrange(5, 80))) for _ in range(8)]
    elif kind == 2: streams = [b"".join(echo_frame(rng, i, (fake * 40)[:rng.choice([100, 1024, 5000])]) for i in range(rng.randrange(5, 60))) for _ in range(8)]
    else: streams = [b"".join(echo_frame(rng, i, rnd62(rng, rng.choice([0, 10, 1024, 30000]))) for i in range(rng.randrange(1, 40))) for _ in range(8)]
    return streams, (ALL if kind in (1, 4) else (1 << 1) | (1 << 2)), kind == 4


def head_entries(rng, runs, true_starts, shift, group, mode):
    """Per tile the speculative entry (only group heads are read): 0 = what a perfect search proposes, 1 = anywhere, 2 = none or a LATER
    true start, 3 = tile edges and one byte past a true start."""
    tile = 1 << shift
    out = []
    for r in range(len(runs)):
        ln = int(runs["length"][r])
        for k in range((ln + tile - 1) >> shift):
            lo, hi = k * tile, min((k + 1) * tile, ln)
            firsts = sorted(p for (rr, p) in true_starts if rr == r and lo <= p < hi)
            if k == 0: e = 0
            elif k % group: e = NONE
            elif mode == 0: e = firsts[0] if firsts else NONE
            elif mode == 1: e = rng.randrange(lo, hi)
            elif mode == 2: e = NONE if rng.random() < 0.5 else (firsts[-1] if firsts else rng.randrange(lo, hi))
            else: e = rng.choice([lo, hi - 1, (firsts[0] + 1) if firsts and firsts[0] + 1 < hi else lo])
            out.append(e)
    return np.array(out or [NONE], np.uint32)


def test_group_walk_resolves_to_the_oracle_and_members_equal_the_per_tile_walk(gw):
    rng = random.Random(SEED + 1201)
    n_cases = n_rew = n_members = 0
    for trial in range(30):
        streams, mask, client = traffic(rng, trial % 5)
        chunks = [s[:rng.randrange(len(s) + 1)] if rng.random() < 0.5 else s for s in streams]
        data, runs = make_runs(chunks)
        runs["preferred_proto"] = rng.choice([-1, 1, 2])
        if client:
            runs["flags"] = 1                                      # B2_RUN_CLIENT: the cut depends on the message before
        rs, msgs, _ = O.process_batch(O.make_config(protocols=mask), data, runs)
        buf = np.concatenate([np.asarray(data, np.uint8), np.zeros(1024, np.uint8)])
        true_starts = set((int(m["run_idx"]), int(m["frame_off"]) - int(runs["offset"][int(m["run_idx"])])) for m in msgs)
        for shift in (9, 11, 13):
            nt = int(sum((int(l) + (1 << shift) - 1) >> shift for l in runs["length"]))
            for group in (2, 4, 8):
                for mode in range(4):
                    entries = head_entries(rng, runs, true_starts, shift, group, mode)
                    rs_d = np.zeros(len(runs), RUN_STATUS_DT); fo = np.zeros(len(msgs) + 64, np.uint32); fr = np.zeros(len(msgs) + 64, np.uint32)
                    nm = C.c_uint32(); rew = C.c_uint32()
                    rc = gw.kh_front_group(buf.ctypes.data, runs.ctypes.data, len(runs), shift, mask, 0, group, entries.ctypes.data, nt,
                                           rs_d.ctypes.data, fo.ctypes.data, fr.ctypes.data, len(fo), C.byref(nm), C.byref(rew))
                    where = (trial, shift, group, mode)
                    assert rc == 0 and nm.value == len(msgs), (where, rc, nm.value, len(msgs))
                    for f in ("consumed", "parse_error", "n_msgs", "first_msg", "preferred_proto"):
                        assert np.array_equal(rs_d[f], rs[f]), (where, f)
                    assert np.array_equal(fo[:nm.value] & 0x7fffffff, msgs["frame_off"]) and np.array_equal(fr[:nm.value], msgs["run_idx"]), where
                    assert np.array_equal(fo[:nm.value] >> 31, (msgs["protocol"] != 1).astype(np.uint32)), where
                    n_cases += 1; n_rew += rew.value
                    recs = np.zeros((max(nt, 1), 5), np.uint32); entered = C.c_uint32()
                    bad = gw.kh_group_vs_tiles(buf.ctypes.data, runs.ctypes.data, len(runs), shift, mask, 0, group, entries.ctypes.data, nt,
                                               recs.ctypes.data, C.byref(entered))
                    assert bad == 0, (where, bad)
                    n_members += entered.value
                    if mode == 0 and not client:
                        # correct heads: a member the walk cut a frame in is entered at a true frame start (an exact continuation of the chain)
                        t = 0
                        for r in range(len(runs)):
                            for k in range((int(runs["length"][r]) + (1 << shift) - 1) >> shift):
                                e, count = int(recs[t, 0]), int(recs[t, 2])
                                assert e == NONE or count == 0 or (r, e) in true_starts, (where, r, k, e)
                                t += 1
    assert n_cases == 30 * 3 * 3 * 4 and n_rew > 500 and n_members > 10000, (n_cases, n_rew, n_members)
