"""CPU: tests/test_gpu_h2_gzip.py, unchanged, on the emulated library (the product's own b2_api.cu / b2_h2.cuh built for the host by
tests/cpp/gen_emul_lib.py, see tests/test_emulated_library.py): the select, size, place and inflate passes of b2_h2_conn_set_gunzip and
their orchestration in b2_h2_process_batch / b2_h2_client_process_batch equal the oracle message for message, and connections without
the opt-in stay byte-identical."""
from test_emulated_library import run_files


def test_gunzip_passes_on_the_emulated_library():
    tail = run_files(["test_gpu_h2_gzip.py"], 1800)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
