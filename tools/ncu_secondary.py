"""Developer tool: launch each secondary kernel once at its perf size so that one `ncu --set full` run captures them all.
usage: ncu --set full --clock-control none -k regex:'ew_kernel|bilateral_kernel|k_light|k_image_loss|k_texel' -o out python tools/ncu_secondary.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import nvdiffrecmc_b200.renderutils as ru
import nvdiffrecmc_b200.optixutils as ou
from nvdiffrecmc_b200.light import EnvironmentLight

dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
B, H, W = 16, 512, 512
t = [torch.rand(B, H, W, 3, generator=g).to(dev).requires_grad_(True) for _ in range(6)]
y = ru.pbr_bsdf(*t)                                                       # ew_kernel<Ew<Pbr, false>>
y.backward(torch.rand_like(y))                                            # ew_kernel<Ew<Pbr, true>>
n = ru.prepare_shading_normal(t[2], t[4], t[0], t[3], t[1], t[5])         # ew_kernel<Ew<Psn, false>>
n.backward(torch.rand_like(n))                                            # ew_kernel<Ew<Psn, true>>
B2 = 8
col = torch.rand(B2, H, W, 3, generator=g).to(dev).requires_grad_(True); col2 = torch.rand(B2, H, W, 3, generator=g).to(dev).requires_grad_(True)
nrm = torch.nn.functional.normalize(torch.rand(B2, H, W, 3, generator=g).to(dev) - 0.5, dim=-1)
zdz = torch.stack([torch.rand(B2, H, W, generator=g).to(dev) + 1, torch.full((B2, H, W), 0.01, device=dev)], -1)
kd = torch.rand(B2, H, W, 3, generator=g).to(dev); ks = torch.rand(B2, H, W, 3, generator=g).to(dev)
out = ou.denoise_and_combine(col, col2, nrm, zdz, 2.0, kd, ks)            # bilateral_kernel<2,0>, ew_kernel<Ew<Combine, false>>
loss = ru.image_loss(out, torch.rand_like(out), loss="l1", tonemapper="log_srgb")     # k_image_loss_fwd
loss.backward()                                                           # k_image_loss_bwd, ew_kernel<Ew<Combine, true>>, bilateral_kernel<2,1>
EnvironmentLight(torch.rand(1024, 2048, 3, generator=g).to(dev))          # k_light_rows, k_light_finish
torch.cuda.synchronize()
print("ok")
