"""Machine-code pins of the DWA and grid planner kernels whose per-robot or per-query body is shared between a
shared-input kernel and a per-agent-input kernel (dwa_robot in crb_dwa.cu; grid_cell_blocked and grid_plan_query in
crb_grid_common.cuh).  The single-map grid kernels are pinned in test_grid_many_maps.py.

crb_dwa_control_many_kernel and crb_dwa_motion_kernel are byte-identical to their code before the body was shared.
crb_dwa_control_kernel and the three many-map grid kernels are not: they have the same instruction count and ptxas
reports the same registers or fewer (crb_dwa_control_kernel 48 where it used 50), no spill and no stack frame, but the
registers are allocated differently.  Their pins hold them from here on."""
from toolchain import kernel_sass_hashes

DWA_SASS = {
    "_Z21crb_dwa_motion_kernellPfPKff": "e2529eb1cc6f6bdcda66adc34f8c1a0eeed167da825c84c8d1225f846c57f389",
    "_Z22crb_dwa_control_kernellPKfPfS0_S0_i14crb_dwa_paramsiS1_PiS1_":
        "1c9f9d5818e823a0c15eb5d0bf4c8b95a4003cea5d40d1365580abaefe30ec01",
    "_Z27crb_dwa_control_many_kernellPKfPfS0_S0_lPKliPKi14crb_dwa_paramsiS1_PiS1_S7_":
        "66e27005dd60a0622c029d4a9421b02a5fcbf8548f21997f1155b59e9b5e6448",
}

GRID_MANY_SASS = {
    "_Z24crb_grid_map_many_kernel11GridMapArgs": "935b00dece1915ebdbb9b10f13dae84546b86e8412eb4fa652f7cff432f5b7aa",
    "_Z25crb_grid_plan_many_kernelILi0EEv16GridPlanManyArgs":
        "64bed61c006e0bca7001ec23f9868ebfb05ab3a81276d85789515a6e9d986865",
    "_Z25crb_grid_plan_many_kernelILi1EEv16GridPlanManyArgs":
        "986a610a293276bc175524ac76aed2e46453d54fe52cbf032071daaa7d0f491a",
}


def test_dwa_kernels_keep_their_machine_code():
    assert kernel_sass_hashes("crb_dwa.cu") == DWA_SASS


def test_many_map_grid_kernels_keep_their_machine_code():
    assert kernel_sass_hashes("crb_grid_many.cu") == GRID_MANY_SASS
