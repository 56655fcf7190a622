"""CPU: tests/test_gpu_h2_serve.py, unchanged, on the emulated library (the product's own b2_api.cu / b2_h2.cuh built for the host by
tests/cpp/gen_emul_lib.py, see tests/test_emulated_library.py): the answering passes of b2_h2_serve_batch (k_h2_serve, the scan,
k_h2_pack on device-built records, the gather) and their orchestration equal the oracle and the twin context reply for reply."""
from test_emulated_library import run_files


def test_serve_passes_on_the_emulated_library():
    tail = run_files(["test_gpu_h2_serve.py"], 1800)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
