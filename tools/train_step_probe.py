"""One Camelyon16-shaped training step (N=15000, C=1; train_tcga.py:67-73,232) for an ncu launch list: which kernels,
how long, and how much of the step is GPU time at all."""
import sys, os, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import dsmil as mil
dev = torch.device('cuda', 0); torch.cuda.set_device(0)
D, NT, CT = 512, 15000, 1
g = torch.Generator(device=dev).manual_seed(7)
tb = [torch.rand(NT, D, generator=g, device=dev) for _ in range(4)]
lab = torch.ones(1, CT, device=dev)
torch.manual_seed(0)
m = mil.MILNet(mil.FCLayer(D, CT), mil.BClassifier(D, CT)).to(dev).train()
opt = torch.optim.Adam(m.parameters(), lr=1e-4, betas=(0.5, 0.9), weight_decay=1e-3)
crit = torch.nn.BCEWithLogitsLoss()
k = [0]
def tstep():
    opt.zero_grad()
    ins, bagp, _, _ = m(tb[k[0] % 4]); k[0] += 1
    mx, _ = torch.max(ins, 0)
    loss = 0.5 * crit(bagp.view(1, -1), lab) + 0.5 * crit(mx.view(1, -1), lab)
    loss.backward()
    opt.step()
steps = int(os.environ.get("PROBE_STEPS", "20"))
ms = bench.cuda_time_ms(tstep, steps, warm=3)
# forward + backward only (no optimizer, no loss glue beyond what autograd needs)
def fb():
    ins, bagp, _, _ = m(tb[0])
    (bagp.sum() + ins.sum()).backward()
ms_fb = bench.cuda_time_ms(fb, steps, warm=3)
with torch.no_grad():
    ms_f = bench.cuda_time_ms(lambda: m(tb[0]), steps, warm=3)
print(json.dumps({"train_step_ms": ms, "fwd_bwd_only_ms": ms_fb, "fwd_train_mode_nograd_ms": ms_f}))
