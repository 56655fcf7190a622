"""GPU: the residency plan of the fused pass on bench.py's shape (64 connections x 4 MiB, 1 KB payloads).  Two contexts on two streams
overlap their passes only if every kernel launched between two k_fused passes can start on an SM that the other batch's 12-warp k_fused
CTA holds; the numbers come from the compiled kernels and the device (b2_resident_plan)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BETWEEN = ("k_tile_search", "k_tile_walk", "k_resolve", "k_pack_slow<true>")


def bench_batch(payload=1024):
    from brpc_b200 import press
    run_bytes = (4 << 20) - 16 * 7
    stride = (run_bytes + 15) // 16 * 16
    data = np.zeros(64 * stride, np.uint8)
    runs, n_full = press.fill_batch(press.spec(payload_bytes=payload), data, 64, run_bytes)
    return data, runs, n_full


def test_pass_kernels_fit_beside_a_12_warp_k_fused():
    import brpc_b200 as b2
    data, runs, n_full = bench_batch()
    ctx = b2.Context(device=0, max_batch_bytes=data.nbytes + (1 << 20), max_msgs=n_full + 4096, max_runs=64,
                     max_resp_bytes=2 * data.nbytes + 96 * n_full + (8 << 20))
    rs, msgs, resp, _ = ctx.process_batch(data, runs)               # (tells the context the frame size, as bench.py's first batch does)
    assert len(msgs) == n_full and np.all(msgs["status"] == 0)
    ctx.upload(data, runs)
    ctx.execute()
    assert ctx.batch_info()["fused"]
    plan = {k["name"]: k for k in ctx.resident_plan()}
    assert set(plan) == {"k_fused", *BETWEEN}
    f = plan["k_fused"]
    assert f["threads"] == 12 * 32 and f["fits"] == 0, f
    for name in BETWEEN:
        k = plan[name]
        assert k["regs"] > 0 and k["threads"] % 32 == 0, k
        assert k["fits"] >= 1, "%s cannot start beside k_fused: %s (k_fused: %s)" % (name, k, f)
    s = plan["k_tile_search"]
    assert s["fits"] * s["threads"] // 32 >= 12, s                  # the speculative search drains 12 warps per SM beside k_fused


def test_dense_shape_leaves_no_room():
    """Small frames (64 B payloads) take k_fused's dense shape (16 warps): what it leaves holds none of the other kernels, and the plan
    says so.  A context that has not finished a batch yet already knows the frame size from the uploaded batch."""
    import brpc_b200 as b2
    data, runs, n_full = bench_batch(payload=64)
    ctx = b2.Context(device=0, max_batch_bytes=data.nbytes + (1 << 20), max_msgs=n_full + 4096, max_runs=64,
                     max_resp_bytes=2 * data.nbytes + 96 * n_full + (8 << 20))
    ctx.upload(data, runs)
    plan = {k["name"]: k for k in ctx.resident_plan()}
    assert plan["k_fused"]["threads"] == 16 * 32
    assert all(plan[name]["fits"] == 0 for name in BETWEEN), plan


def test_first_batch_of_a_context_takes_the_shape_that_leaves_room():
    """bench.py's second context only uploads and launches: its k_fused must already take the 12-warp shape on 1 KB requests."""
    import brpc_b200 as b2
    data, runs, n_full = bench_batch()
    ctx = b2.Context(device=0, max_batch_bytes=data.nbytes + (1 << 20), max_msgs=n_full + 4096, max_runs=64,
                     max_resp_bytes=2 * data.nbytes + 96 * n_full + (8 << 20))
    ctx.upload(data, runs)
    plan = {k["name"]: k for k in ctx.resident_plan()}
    assert plan["k_fused"]["threads"] == 12 * 32
    assert all(plan[name]["fits"] >= 1 for name in BETWEEN), plan
