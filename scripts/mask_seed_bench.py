"""What a region mask costs: masked corner detection on the GPU, and seeding online streams inside object masks.

    python scripts/mask_seed_bench.py [--iters 50] [--steps 12] [--out result.json]

Reports, with the GPU's name and power limit:
  - detect: ms per call and per frame for K = 1, 8 and 64 prepared 384x512 frames in one call, without a mask
    (ct3_detect_corners) and with one disc mask per frame (ct3_detect_corners_masked), and the cost of resizing K
    frame-size 720x1280 masks to 384x512 (ct3_prepare_masks); CUDA events after a warm-up of the same shapes;
  - hub: ms per step of 8 streams of 480x640 chunks (grid 10, history 16) without seeding, with
    seed_corners(sid, 50, mask=...) on every stream before each step, and with the host route a caller has without it
    (frame to the host, cv2.goodFeaturesToTrack with the object mask minus discs around the stream's tracks,
    add_tracks).  The object mask is a disc that moves with the stream.  Each seeded step retires the tracks it added
    afterwards, so every mode tracks the same number of points; a host clock around work that ends in a device
    synchronise.  The cv2 route is reported as not measured when cv2 is not installed.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import corner_cases as C  # noqa: E402
import mask_cases as M  # noqa: E402
from cotracker_b200 import corners, engine  # noqa: E402

DEV = "cuda:0"


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def _time(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_detect(K, iters):
    frames = torch.stack([C.textured_frame(384, 512, seed=s % 8) for s in range(K)]).to(DEV)
    par = corners.params(300, 0.01, 10, 3)
    ws = torch.empty(engine.corners_workspace_bytes(K, 384, 512), dtype=torch.uint8, device=DEV)
    region = torch.stack([torch.from_numpy(M.disc(384, 512, 150 + 8 * (s % 8), 200 + 12 * (s % 8), 120))
                          for s in range(K)]).to(DEV)
    big = torch.stack([torch.from_numpy(M.disc(720, 1280, 300, 500, 220)) for _ in range(K)]).to(DEV)
    plain = _time(lambda: engine.detect_corners(frames, par, workspace=ws), iters)
    masked = _time(lambda: engine.detect_corners(frames, par, workspace=ws, mask=region), iters)
    resize = _time(lambda: engine.prepare_masks(big, (384, 512)), iters)
    n = int(engine.detect_corners(frames, par, workspace=ws)[1][0])
    nm = int(engine.detect_corners(frames, par, workspace=ws, mask=region)[1][0])
    return dict(K=K, ms_per_call=round(plain, 4), ms_per_frame=round(plain / K, 4), masked_ms_per_call=round(masked, 4),
                masked_ms_per_frame=round(masked / K, 4), prepare_masks_720x1280_ms=round(resize, 4),
                corners_frame0=n, masked_corners_frame0=nm)


def bench_hub(mode, steps, cv2=None):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    S, STEP, H, W = 16, 8, 480, 640
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(53, offline=False, window_len=S))
    p = p.to(DEV)
    hub = OnlineStreams(p)
    videos = [texture_video(STEP * (steps + 2) + S, H, W, seed=s, shift=(1 + s % 3, 2)).to(DEV).to(torch.uint8)
              for s in range(8)]
    sids = [hub.open(frame_size=(H, W), grid_size=10, history=16) for _ in videos]
    times = []
    for k in range(steps):
        # each stream's object: a disc of radius 100 drifting with the frame index (a segmenter's output, on the device)
        masks = [torch.from_numpy(M.disc(H, W, 200 + (k * 3 + s) % 80, 260 + (k * 5 + 7 * s) % 120, 100))[None, None]
                 .to(DEV) for s in range(8)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for sid, v in zip(sids, videos):
            hub.push(sid, v[:, STEP * k:STEP * k + S])
        added = {}
        for sid, v, m in zip(sids, videos, masks):
            if mode == "seed":
                added[sid] = hub.seed_corners(sid, 50, min_distance=10, mask=m)
            elif mode == "cv2":
                st = hub._streams[sid]["state"]
                f = v[0, st.length - st.ind].permute(1, 2, 0).cpu().numpy()
                gray = cv2.cvtColor(f, cv2.COLOR_RGB2GRAY)
                mask = (m[0, 0].cpu().numpy() * 255).astype("uint8")
                if st.length:
                    n_keep, scale = hub._streams[sid]["out"]
                    c = st.hist[0][(st.length - 1) % st.hist[0].shape[0], :n_keep].cpu()
                    for x, y in (c * torch.tensor(scale)).tolist():
                        cv2.circle(mask, (int(round(x)), int(round(y))), 12, 0, -1)
                pts = cv2.goodFeaturesToTrack(gray, 50, 0.01, 12, mask=mask)
                if pts is not None:
                    q = torch.from_numpy(pts.reshape(-1, 2)).double()
                    q = torch.cat([torch.full((len(q), 1), float(st.length), dtype=torch.float64), q], 1)[None]
                    added[sid] = hub.add_tracks(sid, q.to(DEV))
        hub.step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        for sid, ids in added.items():
            if ids:
                hub.retire_tracks(sid, ids)
    warm = times[2:]
    return dict(mode=mode, streams=8, frame="480x640", ms_per_step=round(sum(warm) / len(warm), 2),
                min_ms=round(min(warm), 2), steps_timed=len(warm))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_seed_bench.py needs a GPU")
    res = dict(gpu=gpu_info(), detect=[bench_detect(K, a.iters) for K in (1, 8, 64)])
    try:
        import cv2
    except ImportError:
        cv2 = None
    res["hub"] = [bench_hub("none", a.steps), bench_hub("seed", a.steps)]
    res["hub"].append(bench_hub("cv2", a.steps, cv2) if cv2 is not None else dict(mode="cv2", ms_per_step="not measured"))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
