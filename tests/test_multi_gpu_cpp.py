"""The C++-only multi-GPU path (SURVEY §8 b-4): tests/cpp/multi_gpu_demo.cpp drives N GPUs through include/crb.h
alone — one host thread and one crb_ctx per device, libcrb's own NCCL communicator (crb_comm_*), one
crb_gather_stats per call.  CPU: it compiles against the header, links libcrb.so and fails loudly without a GPU.
GPU (needs >= 2 devices, `gpurun --gpus 2`): it runs and every rank gathers the same table."""
import subprocess

import pytest

from cpprobotics_b200 import _lib
from toolchain import build_ref_program


def build(tmp_path):
    return build_ref_program(tmp_path, "multi_gpu_demo.cpp", ("-pthread",))


def test_compiles_links_and_needs_a_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: the failure path is covered on the CPU box")
    r = subprocess.run([exe, "2", "64"], capture_output=True, text=True)
    assert r.returncode == 3 and "no CPU fallback" in r.stderr


def test_nccl_is_found_at_run_time():
    # dlopen'ed, not linked: libcrb.so itself must not depend on libnccl
    out = subprocess.check_output(["ldd", _lib.LIB_PATH], text=True)
    assert "nccl" not in out
    assert _lib.load_library().crb_comm_nccl_version() >= 22000


@pytest.mark.gpu
def test_two_gpus_from_cpp(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (gpurun --gpus 2)")
    exe = build(tmp_path)
    world = min(torch.cuda.device_count(), 8)
    r = subprocess.run([exe, str(world), "16384"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "multi_gpu_demo OK" in r.stdout
