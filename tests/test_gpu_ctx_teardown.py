"""GPU: destroying a context gives back every device buffer it reserved, so a training run that creates and drops contexts does not
leak device memory."""
import pytest
import torch

from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def test_create_build_destroy_returns_device_memory(dev):
    import nvdiffrecmc_b200.optixutils as ou
    small = [torch.tensor(a, device=dev) for a in synth.scene_mesh("blob+torus", level=4)]   # 7 168 triangles: SAH shadow view
    large = [torch.tensor(a, device=dev) for a in synth.scene_mesh("grid1m", level=0)]       # 1.08 M triangles: LBVH shadow view
    # The baseline is taken before the first context: the stream-ordered pool returns memory in whole chunks (32 MB on an H100), so
    # after a warm-up cycle a leaked buffer would pin a chunk the baseline already counts, and later leaks would fit inside it.
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for i in range(100):
        ctx = ou.OptiXContext()
        for v, f in ([small, large] if i % 25 == 0 else [small]):   # small then large: every buffer grows, both shadow views allocate
            ou.optix_build_bvh(ctx, v, f, rebuild=1)
        del ctx                                                     # synchronises, then destroys the context
    torch.cuda.synchronize()
    lost = free0 - torch.cuda.mem_get_info()[0]
    assert lost < 2 << 20, "%.1f MB of device memory not returned after 100 contexts" % (lost / 2**20)
