"""A small, fast pass over every hand-written kernel for compute-sanitizer (memcheck / synccheck / racecheck are
10-100x slower than native, so the shapes are tiny).  Each case also checks its result against the CPU oracle.
    compute-sanitizer --tool memcheck  python tests/tools/sanitize_cases.py > profiles/r2_sanitizer_memcheck.log
    compute-sanitizer --tool synccheck python tests/tools/sanitize_cases.py > profiles/r2_sanitizer_synccheck.log"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cotracker_b200 import engine as eng  # noqa: E402
from cotracker_b200.build import build_cotracker  # noqa: E402
from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video  # noqa: E402
from oracle import ct3_oracle as O  # noqa: E402

DEV = "cuda:0"


def corr_stage():
    T, N, H4, W4 = 3, 40, 64, 72
    g = torch.Generator().manual_seed(2)
    fmaps = torch.randn(T, 128, H4, W4, generator=g) * 2.5
    want_pyr = O.normalized_pyramid(fmaps)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    support = torch.randn(4, 49, N, 128, generator=g)
    support = support / support.norm(dim=-1, keepdim=True)
    coords = torch.rand(T, N, 2, generator=g) * torch.tensor([W4 + 6.0, H4 + 6.0]) - 3.0
    valid = torch.ones(N, dtype=torch.uint8)
    for impl, corr, fc1 in ((0, 2, 3), (0, 1, 2), (0, 3, 3), (2, 3, 3), (1, 3, 3)):
        eng.set_option("corr", impl); eng.set_option("prec.corr", corr); eng.set_option("prec.fc1", fc1)
        got = eng.corr_sample(pyr, H4, W4, support.to(DEV), valid.to(DEV), coords.to(DEV)).cpu()
        err = max(float((got[:, :, l].permute(1, 0, 2) - O.correlation_volume(want_pyr[l], support[l], coords / 2 ** l)).abs().max())
                  for l in range(4))
        print(f"corr impl={impl} prec.corr={corr} prec.fc1={fc1}: max err {err:.2e}")
        assert err < 5e-4
    eng.set_option("corr", 0); eng.set_option("prec.corr", 2); eng.set_option("prec.fc1", 3)


def model_cases():
    sd = seeded_state_dict(11, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)
    video = texture_video(4, 256, 288, seed=3)
    queries = random_queries(80, 4, 256, 288, seed=4)   # > 64 points: point<-virtual attention over many tiles
    with torch.no_grad():
        want_c, want_v, _ = O.offline_forward(sd, video, queries, iters=2)
    model = build_cotracker(None, offline=True, window_len=60).eval()
    model.load_state_dict(sd)
    model = model.to(DEV)
    for fuse, attn in ((1, 0), (0, 0)):
        eng.set_option("fuse", fuse); eng.set_option("attn", attn)
        c, v, q, _ = model(video.to(DEV), queries.to(DEV), iters=2)
        torch.cuda.synchronize()
        err = float((c.cpu() - want_c).abs().max())
        print(f"model (encoder + loop) fuse={fuse} attn={attn}: max |d tracks| {err:.2e} px")
        assert err < 1e-3
    eng.set_option("fuse", 1); eng.set_option("attn", 0)


if __name__ == "__main__":
    corr_stage()
    model_cases()
    print("sanitize_cases: all cases ran")
