"""EKF step code generation and the access-pattern probe.
CPU: the two EKF kernels the launcher selects compile for sm_90a, with the build's flags, without spilling to
local memory.  H100: the two-agent form of the step (even n, 8-byte aligned arrays) gives the same bits as the
one-agent form, over several steps per launch; crb_probe_ekf_pattern does what include/crb.h says it does."""
import numpy as np
import pytest

from cpprobotics_b200 import synth
from toolchain import ptxas_kernels


def test_ekf_compiles_only_the_two_launch_forms_without_spill():
    kernels = {k: f for k, f in ptxas_kernels("crb_ekf.cu").items() if "crb_ekf_step" in k}
    # the two-agent form <128,4,2> and the one-agent form <256,3,1>
    assert set(kernels) == {"_Z19crb_ekf_step_kernelILi128ELi4ELi2EEvllPfS0_PKfS2_li7EkfArgs",
                            "_Z19crb_ekf_step_kernelILi256ELi3ELi1EEvllPfS0_PKfS2_li7EkfArgs"}, sorted(kernels)
    for f in kernels.values():
        assert (f.spill_stores, f.spill_loads) == (0, 0), f


@pytest.mark.gpu
@pytest.mark.parametrize("n_steps", [1, 3])
def test_ekf_two_agent_form_is_bitwise_the_one_agent_form(engine, n_steps):
    """n = 20_001 is odd, so its launch takes the one-agent kernel; its first 20_000 agents run again as an even
    batch, which takes the two-agent kernel.  Agents are independent, so the bits must agree."""
    import torch
    n = 20_001
    x, P, z, u = synth.ekf_inputs(n, n_steps=n_steps)
    odd = [torch.from_numpy(a).cuda() for a in (x, P, z, u)]
    even = [torch.from_numpy(np.ascontiguousarray(a[:, : n - 1])).cuda() for a in (x, P, z, u)]
    engine.ekf_estimation(*odd, n_steps=n_steps)
    engine.ekf_estimation(*even, n_steps=n_steps)
    torch.cuda.synchronize()
    assert np.array_equal(odd[0].cpu().numpy()[:, : n - 1], even[0].cpu().numpy())
    assert np.array_equal(odd[1].cpu().numpy()[:, : n - 1], even[1].cpu().numpy())


@pytest.mark.gpu
def test_ekf_pattern_probe_adds_the_agent_sum(engine):
    import torch
    n = 100_002
    x, P, z, u = synth.ekf_inputs(n)
    t = [torch.from_numpy(a).cuda() for a in (x, P, z, u)]
    engine.probe_ekf_pattern(*t)
    torch.cuda.synchronize()
    s = (z[0] + z[1]) + (u[0] + u[1])
    assert np.array_equal(t[0].cpu().numpy(), x + s) and np.array_equal(t[1].cpu().numpy(), P + s)
    assert np.array_equal(t[2].cpu().numpy(), z) and np.array_equal(t[3].cpu().numpy(), u)
