"""CPU: tests/test_gpu_h2_client_rx.py, unchanged, on the emulated library (the product's own b2_api.cu / b2_h2.cuh built for the host by
tests/cpp/gen_emul_lib.py, see tests/test_emulated_library.py): the client kernel's data flow and the host orchestration of
b2_h2_client_conn_reset / b2_h2_pack_requests / b2_h2_client_process_batch / b2_h2_client_abandon_streams equal the oracle call for call,
on the recorded grpcio conversation split at many offsets, the hand-built frames, the pool limits and a live grpcio round trip."""
from test_emulated_library import run_files


def test_client_receive_path_on_the_emulated_library():
    tail = run_files(["test_gpu_h2_client_rx.py"], 1800)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
