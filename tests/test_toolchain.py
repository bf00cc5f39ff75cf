"""CPU: the ptxas -v report is read per function, so a kernel's stack frame and spills are its own, never those of an
out-of-line function listed after it."""
from toolchain import PtxasFunction, parse_ptxas

# CUDA 12.9's ptxas -v for crb_pf.cu and crb_pf_fleet.cu, cut down to two kernels
REPORT = """\
ptxas info    : Compiling entry function '_Z21crb_pf_gather2_kerneliPKfPKdS2_S2_ifS0_jjPfS3_PdS2_d' for 'sm_90a'
ptxas info    : Function properties for _Z21crb_pf_gather2_kerneliPKfPKdS2_S2_ifS0_jjPfS3_PdS2_d
    24 bytes stack frame, 16 bytes spill stores, 24 bytes spill loads
ptxas info    : Used 32 registers, used 1 barriers, 24 bytes cumulative stack size, 28876 bytes smem
ptxas info    : Compile time = 285.143 ms

ptxas info    : 24 bytes gmem
ptxas info    : Compiling entry function '_Z19crb_pf_fleet_kernelPfS_S_PKfS1_S1_PKlPKiS1_PdPi11PfFleetArgs' for 'sm_90a'
ptxas info    : Function properties for _Z19crb_pf_fleet_kernelPfS_S_PKfS1_S1_PKlPKiS1_PdPi11PfFleetArgs
    32 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads
ptxas info    : Used 80 registers, used 0 barriers, 32 bytes cumulative stack size
ptxas info    : Compile time = 414.731 ms
ptxas info    : Function properties for _ZN46_INTERNAL_0671617b_15_crb_pf_fleet_cu_98c7cc3724crb_sincosf_reduce_largeEf
    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads
"""


def test_each_function_has_its_own_record():
    assert parse_ptxas(REPORT) == [
        PtxasFunction("_Z21crb_pf_gather2_kerneliPKfPKdS2_S2_ifS0_jjPfS3_PdS2_d", True, 32, 24, 16, 24),
        PtxasFunction("_Z19crb_pf_fleet_kernelPfS_S_PKfS1_S1_PKlPKiS1_PdPi11PfFleetArgs", True, 80, 32, 0, 0),
        PtxasFunction("_ZN46_INTERNAL_0671617b_15_crb_pf_fleet_cu_98c7cc3724crb_sincosf_reduce_largeEf", False, None,
                      0, 0, 0),
    ]
