"""The 3xFP16 / 3xTF32 projection kernel (gemm3x_kernel, csrc/wgmma.cuh) runs one k-block ahead across tile boundaries:
while a k-block's wgmma group runs it waits for the next stage of the ring -- k-block 0 of the CTA's next tile after a
tile's last k-block -- and splits its fragments, and it issues the next tile's first group before the finished tile's
epilogue.  These cases make a CTA cross many tile boundaries with the ring in every relative position: one k-block per
tile (every k-block is a boundary), as many k-blocks as ring stages (each tile's k-block 0 lands in the slot of the
previous tile's k-block 0) and one more than that, on grids capped at 1, 2 and 5 CTAs and tiles - 1.  Every instance must
stay within its float64 bound and give the bits of the uncapped grid (one tile per CTA)."""
import pytest
import torch

from test_gemm_paths import C_OF, DEV, INSTANCES, check_bound, make_w, run_instance

STAGES = {True: 3, False: 4}  # ring depth of the fp16 / TF32 forms (Gemm3xShape::kStages)
K_BLOCK = {True: 64, False: 32}


@pytest.fixture(scope="module")
def cabi():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p.cabi


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES)
def test_tile_boundaries_on_capped_grids(cabi, inst):
    g = torch.Generator().manual_seed(21)
    f16 = inst.startswith("f16")
    M, N = 600, 300  # 5 x 3 = 15 tiles
    tiles = 15
    for i, kblocks in enumerate((1, STAGES[f16], STAGES[f16] + 1)):
        K = kblocks * K_BLOCK[f16]
        act = 0 if inst == "f16_scaled" else i % 3
        x = torch.randn(M, K, generator=g).to(DEV)
        w, b = make_w(("randn", "wide")[i % 2], N, K, g).to(DEV), torch.randn(N, generator=g).to(DEV)
        want, a_s, w_s = run_instance(cabi, inst, x, w, b, act)
        check_bound(inst, want, x, w, b, act, C_OF[inst], a_s, w_s)
        try:
            for cap in (1, 2, 5, tiles - 1):
                cabi.lib().sdetr_set_persistent_ctas(cap)
                assert torch.equal(run_instance(cabi, inst, x, w, b, act)[0], want), (inst, kblocks, cap)
        finally:
            cabi.lib().sdetr_set_persistent_ctas(0)
