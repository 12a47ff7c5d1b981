"""Experiment: where does the ResNet-18-InstanceNorm embedder spend its time, and would channels_last help?"""
import os, sys, json
import torch, torchvision.models as models
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
dev = torch.device('cuda', 0)
torch.cuda.set_device(0)
x = torch.rand(128, 3, 224, 224, device=dev)

class Id(torch.nn.Module):
    def __init__(self, *a, **k): super().__init__()
    def forward(self, x): return x

def mk(norm):
    torch.manual_seed(0)
    m = models.resnet18(weights=None, norm_layer=norm); m.fc = torch.nn.Identity()
    return m.to(dev).eval()
out = {}
with torch.no_grad():
    for name, norm in (("instnorm", torch.nn.InstanceNorm2d), ("no_norm", Id)):
        m = mk(norm)
        out[name + "_nchw_ms"] = bench.cuda_time_ms(lambda: m(x), 5, warm=2)
        m2 = mk(norm).to(memory_format=torch.channels_last); xc = x.contiguous(memory_format=torch.channels_last)
        out[name + "_nhwc_ms"] = bench.cuda_time_ms(lambda: m2(xc), 5, warm=2)
    torch.backends.cudnn.benchmark = True
    for name, norm in (("no_norm_bench", Id),):
        m = mk(norm)
        out[name + "_nchw_ms"] = bench.cuda_time_ms(lambda: m(x), 5, warm=3)
        m2 = mk(norm).to(memory_format=torch.channels_last); xc = x.contiguous(memory_format=torch.channels_last)
        out[name + "_nhwc_ms"] = bench.cuda_time_ms(lambda: m2(xc), 5, warm=3)
    torch.backends.cudnn.benchmark = False
    import dsmil as mil
    from dsmil_wsi_b200.embedder import fuse_instance_norm
    m = mk(torch.nn.InstanceNorm2d); fuse_instance_norm(m)
    out["instnorm_fused_nchw_ms"] = bench.cuda_time_ms(lambda: m(x), 5, warm=2)
    # bf16 autocast convs for scale (not a parity candidate)
    m = mk(Id).to(memory_format=torch.channels_last)
    with torch.autocast('cuda', dtype=torch.bfloat16):
        out["no_norm_nhwc_bf16_ms"] = bench.cuda_time_ms(lambda: m(xc), 5, warm=2)
print(json.dumps(out, indent=1))
