"""CPU: tests/test_gpu_streams.py, unchanged, on the emulated library (the product's own b2_api.cu / b2_kernels.cuh built for the host by
tests/cpp/gen_emul_lib.py, see tests/test_emulated_library.py): the stream pass — k_stream_route / alloc / group / run / rst behind k_small and
behind the big pipeline, the host-side table calls and the result plumbing — equals the oracle.  The lanes of a warp are host threads that the
scheduler interleaves freely here, so a walk that relies on the warp staying converged shows as wrong bytes."""
from test_emulated_library import run_files


def test_stream_pass_on_the_emulated_library():
    tail = run_files(["test_gpu_streams.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
