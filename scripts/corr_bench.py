"""Correlation stage alone at the headline size (N=6400, T=16, 96x128 feature maps): ms per launch, CUDA events.
    CT3_B200_LIB=<variant .so> python scripts/corr_bench.py [impl [prec.corr [prec.fc1]]]
impl is the "corr" option: 0 correlate-then-interpolate (corr_tc3.cu for prec.corr 1 | 2, corr_tc2.cu for 3), 1 exact-fp32
SIMT, 2 sample-then-correlate (corr_tc.cu)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from cotracker_b200 import engine

impl = int(sys.argv[1]) if len(sys.argv) > 1 else 0
dev = "cuda:0"
T, N, H4, W4 = 16, 6400, 96, 128
g = torch.Generator().manual_seed(0)
fmaps = torch.randn(T, 128, H4, W4, generator=g).to(dev)
pyr = engine.prepare_pyramid(fmaps)
support = torch.randn(4, 49, N, 128, generator=g).to(dev)
base = torch.rand(1, N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])
coords = (base + torch.randn(T, N, 2, generator=g) * 2.0).to(dev).contiguous()
vol = torch.empty(N * T * 4, 2 * 2432, dtype=torch.bfloat16, device=dev)
scr = torch.empty(pyr.numel() * 4, dtype=torch.uint8, device=dev)
engine.set_option("corr", impl)
if len(sys.argv) > 2:
    engine.set_option("prec.corr", int(sys.argv[2]))
if len(sys.argv) > 3:
    engine.set_option("prec.fc1", int(sys.argv[3]))
lib = engine.lib()
def run():
    rc = lib.ct3_corr_sample(pyr.data_ptr(), H4, W4, support.data_ptr(), None, coords.data_ptr(), T, N, vol.data_ptr(),
                             scr.data_ptr(), scr.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.ct3_last_error()
for _ in range(3):
    run()
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(11)]
for i in range(10):
    ev[i].record(); run()
ev[10].record(); torch.cuda.synchronize()
ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(10))
print(f"{os.environ.get('CT3_B200_LIB', 'default')} impl={impl} prec={sys.argv[2:]}: corr_sample (+pyramid split) median {ms[5]:.3f} ms, min {ms[0]:.3f} ms")
