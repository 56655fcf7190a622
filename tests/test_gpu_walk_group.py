"""GPU: walk groups of the front stages (b2_set_walk_group, DESIGN §3).  The same batches run with one tile per group, 2, 4 and 8 tiles
per group, and the automatic choice; run statuses, descriptors and every reply byte must be the oracle's every time.  Each context runs
its batch twice: the first pass learns the frame size from the batch, the second follows what the first one saw (the fused path, or the
slot-scan pipeline after a batch heavy in slow replies).  On the emulated library (tests/emul_runner.py) the batches are smaller."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import _oracle as O  # noqa: E402
from _compare import assert_same  # noqa: E402
from _traffic import SEED, echo_frame, mixed_frames, rnd62  # noqa: E402

EMUL = bool(os.environ.get("B2_EMUL_LIB"))
MODES = (1, 2, 4, 8, 0)                     # 0 = auto
ALL = (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4) | (1 << 12)


@pytest.fixture(scope="module")
def b2():
    import brpc_b200
    return brpc_b200


def press_batch(n_sockets, run_bytes, payload, checksum=0):
    from brpc_b200 import press
    data = np.zeros(n_sockets * ((run_bytes + 15) // 16 * 16), np.uint8)
    runs, _ = press.fill_batch(press.spec(payload_bytes=payload, payload_kind=1, checksum_type=checksum), data, n_sockets, run_bytes)
    return data, runs


def run_modes(b2, data, runs, protocols=None, what=""):
    """Every mode, twice each, against the oracle; returns the group size each mode's second launch used."""
    orc = O.process_batch(O.make_config(protocols=protocols) if protocols else O.make_config(), data, runs)
    used = {}
    for mode in MODES:
        ctx = b2.Context(device=0, max_batch_bytes=data.nbytes + (1 << 20), max_msgs=len(orc[1]) + 4096, max_runs=max(64, len(runs)),
                         max_resp_bytes=2 * data.nbytes + 96 * len(orc[1]) + (8 << 20))
        if protocols:
            ctx.set_protocols(protocols)
        ctx.set_walk_group(mode)
        for rep in range(2):
            dev = ctx.process_batch(data, runs)
            assert_same(dev, orc, "%s mode %d pass %d (group %d, fused %d)" % (what, mode, rep, ctx.walk_group(), ctx.batch_info()["fused"]))
            if mode >= 2:
                assert ctx.walk_group() == mode, (what, mode, ctx.walk_group())
        used[mode] = (ctx.walk_group(), ctx.batch_info()["fused"])
    assert used[1][0] == 1
    return used


@pytest.mark.parametrize("payload", [64, 1024, 4096, 65536])
def test_payload_sizes(b2, payload):
    run_bytes = (1 << 20) if EMUL else (4 << 20)
    if payload == 65536 and not EMUL:
        run_bytes = 8 << 20                 # (64 KiB frames take 512 KiB tiles: several groups per connection)
    data, runs = press_batch(4 if EMUL else 16, run_bytes - 77, payload)
    used = run_modes(b2, data, runs, what="payload %d" % payload)
    if payload >= 1024:
        assert used[0] == (2, 1), used      # auto: 2 tiles per group on the fused path once the frame size is known
    else:
        assert used[0][0] == 1, used        # small frames take the dense shape: one tile per group


def test_crc32c_requests(b2):
    data, runs = press_batch(4 if EMUL else 16, (1 << 20) - 77, 1024, checksum=1)
    run_modes(b2, data, runs, what="crc32c")


def test_payloads_that_are_frame_chains(b2):
    """Payloads carrying whole frames: a wrong group head walks a chain of look-alikes across its members, which k_resolve re-walks."""
    rng = random.Random(SEED + 1301)
    fake = b"".join(echo_frame(rng, i, b"y" * rng.choice([20, 300, 1100])) for i in range(40))
    n, per = (6, 120) if EMUL else (32, 1500)
    chunks = [b"".join(echo_frame(rng, i, fake[rng.randrange(64):][:rng.choice([100, 1024, 5000])]) for i in range(per)) for _ in range(n)]
    chunks = [c[:len(c) - rng.randrange(200)] for c in chunks]
    data, runs = b2.make_runs(chunks)
    run_modes(b2, data, runs, what="frame chains")


def test_mixed_protocol_masks(b2):
    """Five-protocol traffic with garbage on server runs, and client runs with every handler enabled (their cut depends on the message before)."""
    from test_core_cut_host import five_protocol_stream
    rng = random.Random(SEED + 1302)
    n, per = (6, 60) if EMUL else (24, 600)
    for client in (False, True):
        chunks = [b"".join(five_protocol_stream(rng, per)) for _ in range(n)]
        data, runs = b2.make_runs(chunks)
        if client:
            runs["flags"] = 1                                              # B2_RUN_CLIENT
        run_modes(b2, data, runs, protocols=ALL, what="five protocols client=%d" % client)
    chunks = [b"".join(mixed_frames(rng, per, big=rng.random() < 0.3)) for _ in range(n)]
    data, runs = b2.make_runs(chunks)
    run_modes(b2, data, runs, what="mixed frames")


def test_bench_shape(b2):
    """bench.py's batch: 64 connections x 4 MiB of 1 KB requests, each run cut mid-frame."""
    n, run_bytes = (8, 1 << 20) if EMUL else (64, 4 << 20)
    data, runs = press_batch(n, run_bytes - 16 * 7, 1024)
    used = run_modes(b2, data, runs, what="bench shape")
    assert used[0] == (2, 1), used


def test_walk_group_mode_is_checked(b2):
    ctx = b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=8)
    with pytest.raises(b2.B2Error):
        ctx.set_walk_group(9)
