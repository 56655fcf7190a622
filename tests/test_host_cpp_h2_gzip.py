"""GPU: b2::GpuH2Messenger with SetGunzip(true) (brpc_b200/host/h2_messenger.h) — builds tests/cpp/h2_gzip_messenger_test with g++ and
runs it: gzip-compressed gRPC echo requests are inflated on the device and echoed from the device's out buffer, every byte written back
identical to the oracle (C oracle parse and reply framing, request inflated by its GzipInputStream)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "h2_gzip_messenger_test")


@pytest.mark.gpu
def test_gpu_h2_messenger_gunzip_cpp():
    import brpc_b200  # noqa: F401  (the library is built)
    import _oracle  # noqa: F401  (the oracle library is built)
    src = os.path.join(ROOT, "tests", "cpp", "h2_gzip_messenger_test.cc")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-o", BIN, src,
                           "-L" + os.path.join(ROOT, "brpc_b200"), "-lb2rpc", "-L" + os.path.join(ROOT, "oracle"), "-loracle",
                           "-Wl,-rpath," + os.path.join(ROOT, "brpc_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "h2 gunzip messenger ok" in out.stdout
