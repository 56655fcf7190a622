"""CPU: tests/test_gpu_walk_group.py, unchanged, on the emulated library (see tests/test_emulated_library.py): every walk group mode
against the oracle, plain and with asynchronous copies landing as late as the waits allow."""
from test_emulated_library import run_files


def test_walk_groups_on_the_emulated_library():
    tail = run_files(["test_gpu_walk_group.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail


def test_walk_groups_with_late_asynchronous_copies():
    tail = run_files(["test_gpu_walk_group.py"], 3000, B2_EMUL_ASYNC="late")
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
