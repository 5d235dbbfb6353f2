"""Debug helper (not a test): per-parameter gradient error table of the synthesis backward."""
import importlib, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from oracle import port
pkg = importlib.import_module("3dhumangan_b200")
st = importlib.import_module("3dhumangan_b200.modules.synthesis_train")
C = 256
cfg = pkg.configs.baseline_config("tiny")
cfg.update(gen_height=16, gen_width=24, mod_blocks=[], map3d_mode="mixed")
B, Hg, Wg = 2, cfg["gen_height"], cfg["gen_width"]
params = port.init_generator_params(cfg, seed=5)
names = [n for n in params if n.startswith(("synthesis_network.", "synthesis_input."))]
learn = [n for n in names if not n.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked"))]
g = torch.Generator().manual_seed(6)
fixed = torch.randn(B, 1, C, generator=g) * 0.5
wgt = torch.randn(B, 3, Hg, Wg, generator=g)
pc = {n: params[n].clone().double() if params[n].is_floating_point() else params[n].clone() for n in names}
for n in learn:
    pc[n].requires_grad_(True)
fc = fixed.clone().double().requires_grad_(True)
x0 = port.synthesis_input(pc, B, Hg, Wg) if False else torch.sin(torch.nn.functional.conv2d(
    torch.stack([torch.linspace(-1, 1, Hg).double()[:, None].expand(Hg, Wg), torch.linspace(-1, 1, Wg).double()[None, :].expand(Hg, Wg)], 0)[None].repeat(B, 1, 1, 1),
    pc["synthesis_input.network.0.weight"], pc["synthesis_input.network.0.bias"]))
pg = {n: params[n].clone().cuda() for n in names}
for n in learn:
    pg[n].requires_grad_(True)
rgb, tape = st.synthesis_forward_train(pg, None, fixed.cuda(), cfg)
# LeakyReLU masks of OUR forward (the gradient is discontinuous in them): the fp64 reference below uses the same
masks = []
HW = Hg * Wg
for rec in tape.halves:
    x = rec["x"][0].expand(B, -1, -1, -1)          # one 256-channel half; the synthesis input is batch-shared
    xp = x.permute(0, 2, 1, 3).reshape(B, C, -1)[:, :, :HW].double().cpu()
    m = rec["mod_d"][0].double().cpu()
    pre = xp * m[:, 0, :, None] + m[:, 1, :, None]
    masks.append(torch.where(pre > 0, 1.0, 0.2).reshape(B, C, Hg, Wg))
if "--samemask" in sys.argv:
    it = iter(masks)
    port.F = type("Fpatched", (), {k: getattr(torch.nn.functional, k) for k in dir(torch.nn.functional)})
    port.F.leaky_relu = staticmethod(lambda v, slope: v * next(it))
rgb_ref = port.synthesis_network(pc, x0, torch.zeros(B, C, Hg, Wg).double(), fc, cfg, training=True)
(rgb_ref * wgt.double()).sum().backward()
print("fwd err", float((rgb.cpu().double() - rgb_ref.detach()).abs().max() / rgb_ref.abs().max()))
dfs = st.synthesis_backward(pg, tape, wgt.cuda())
torch.cuda.synchronize()
rows = []
for n in learn:
    if pc[n].grad is None:
        continue
    a, b = pg[n].grad.cpu().double(), pc[n].grad.double()
    rows.append(((a - b).norm().item() / max(b.norm().item(), 1e-30), b.norm().item(), (a - b).norm().item(), n))
for r in rows:
    print("%.3e  |ref| %.3e  |diff| %.3e  %s" % r)
print("fixed_style", float((dfs.cpu().double().reshape(-1) - fc.grad.reshape(-1)).norm() / fc.grad.norm()))
