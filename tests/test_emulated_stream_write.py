"""CPU: tests/test_gpu_stream_write.py, unchanged, on the emulated library (the product's own b2_api.cu / b2_kernels.cuh built for the host
by tests/cpp/gen_emul_lib.py, see tests/test_emulated_library.py): b2_stream_write — k_sw_route / alloc / group / admit / scan / frames /
copy, the host-side checks and staging, FROM_MSG reads of the last batch and the WRITABLE events of the stream pass — equals the oracle.
The lanes of a warp are host threads that the scheduler interleaves freely here, so a walk that relies on the warp staying converged
shows as wrong bytes."""
from test_emulated_library import run_files


def test_stream_write_on_the_emulated_library():
    tail = run_files(["test_gpu_stream_write.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
