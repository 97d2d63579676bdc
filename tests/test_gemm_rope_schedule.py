"""The QKV projection's 256-channel RoPE instance computes, bit for bit, what the 128-channel RoPE instance computes.

The wide instance (gemm_wgmma_kernel<256, EM_ROPE, 0>, gemm_tc.cu) gives each CTA a contiguous range of 128-frame x
256-channel tiles, keeps the A rows of the current 128-frame block resident in shared memory and hands 128-channel
half-tiles to its two consumer warpgroups in turn.  The MMA shape, the k order and the epilogue's floating-point
operations are those of the 128-channel instance, so the q / k / v planes must match exactly.  The grids below make CTA
ranges start in the middle of a frame block and cross frame blocks; a huge SM-count override forces 128-channel tiles
for the reference run, as the wide instance runs only when there are at least as many tiles as SMs."""
import pytest
import torch

from kernel_harness import bits, run_ok
from kernel_harness import dev, handles  # noqa: F401 (fixtures)
from test_gemm_contract import BIAS, H, ROPE, make_tensors, problem, run_hook

GRIDS = (1, 2, 5, 7, 131, 132)
NARROW = 1 << 20                    # an SM count no problem here has as many tiles as: 128-channel tiles


@pytest.mark.gpu
@pytest.mark.parametrize("BB", [1, 4, 64])
@pytest.mark.parametrize("T", [1, 129, 1000])
def test_wide_rope_matches_narrow_bit_for_bit(BB, T, dev, handles):
    lib, hs = handles
    d = problem(B=max(1, BB // 2), BB=BB, T=T, C0=H, N=3 * H, flags=BIAS | ROPE, rope_H=H, planes=True, ksplit=1)
    t = make_tensors(d, 90 + BB + T)
    ref, plan = run_ok(run_hook, lib, hs["tc"], dict(d, num_sms=NARROW), t, dev)
    assert plan.bn == 128
    assert not torch.isnan(ref["out"]).any()
    tiles = BB * -(-T // 128) * (3 * H // 256)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    grids = sorted({g for g in GRIDS + (sms,) if g <= tiles})
    for g in grids:
        o, plan = run_ok(run_hook, lib, hs["tc"], dict(d, num_sms=g), t, dev)
        assert plan.bn == 256 and plan.grid == g, (g, plan.bn, plan.grid)
        for k in ref:
            assert torch.equal(bits(o[k]), bits(ref[k])), (g, k)
