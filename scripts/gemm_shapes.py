"""Time every GEMM shape of the headline step (512^2 x 16 frames, grid 80: N = 6400 tracks, T = 16, 6 iterations) on
the tensor-core GEMM through ct3_linear_prec, one shape at a time:

    python scripts/gemm_shapes.py [--seconds 1.0]

Operands are split into 16-bit planes once, outside the timed region; each shape is then launched back to back for at
least --seconds between two CUDA events.  Prints the card, its power limit and max SM clock, then per shape the time
per launch, the algorithmic TFLOP/s (2*M*N*K with the true K) and the launches per iteration, and at the end the GEMM
time per step that these shapes add up to (the time-block q|k|v projection runs in the fused attention kernel and is
not included).  The fp32 output epilogue stands in for each layer's own (split-bf16 stores, residual adds).
CT3_B200_LIB selects the library build to time."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cotracker_b200 import engine  # noqa: E402

ITERS = 6
N, T, V = 6400, 16, 64
RP, RV = N * T, V * T                   # point-token rows, virtual-token rows
RA, MC = RP + RV, RP * 4                # all token rows (time blocks), correlation-MLP rows (4 levels)

# (layers, M, N, K, act, products, fp16 planes, launches per iteration); act 1 = GELU(erf), 2 = GELU(tanh)
SHAPES = [
    ("corr_mlp.fc1 (fp16 planes)", MC, 384, 2401, 1, 3, True, 1),
    ("corr_mlp.fc1 (bf16 planes)", MC, 384, 2401, 1, 3, False, 0),
    ("corr_mlp.fc2", MC, 256, 384, 0, 3, False, 1),
    ("input_transform", RP, 384, 1110, 0, 3, False, 1),
    ("time out", RA, 384, 384, 0, 3, False, 3),
    ("time mlp.fc1", RA, 1536, 384, 2, 3, False, 3),
    ("time mlp.fc2", RA, 384, 1536, 0, 3, False, 3),
    ("point q, out", RP, 384, 384, 0, 3, False, 6),
    ("point kv", RP, 768, 384, 0, 3, False, 3),
    ("point mlp.fc1", RP, 1536, 384, 2, 3, False, 3),
    ("point mlp.fc2", RP, 384, 1536, 0, 3, False, 3),
    ("virtual q, out", RV, 384, 384, 0, 3, False, 9),
    ("virtual kv", RV, 768, 384, 0, 3, False, 3),
    ("virtual qkv", RV, 1152, 384, 0, 3, False, 3),
    ("virtual mlp.fc1", RV, 1536, 384, 2, 3, False, 6),
    ("virtual mlp.fc2", RV, 384, 1536, 0, 3, False, 6),
]


def card(dev):
    q = subprocess.run(["nvidia-smi", f"--id={dev}", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(dev) + " (nvidia-smi failed)"


def time_shape(M, Nout, K, act, products, fp16, seconds, dev):
    Kpad = (K + 63) // 64 * 64
    g = torch.Generator(device=dev).manual_seed(M + Nout + K)
    xs = engine.split_rows(torch.randn(M, K, device=dev, generator=g), Kpad, fp16)
    ws = engine.split_rows(torch.randn(Nout, K, device=dev, generator=g) * K ** -0.5, Kpad, fp16)
    bias = torch.randn(Nout, device=dev, generator=g)
    y = torch.empty(M, Nout, dtype=torch.float32, device=dev)
    lib, stream = engine.lib(), engine._stream(dev)
    args = (engine._ptr(xs), engine._ptr(ws), engine._ptr(bias), M, Nout, Kpad, act, products, int(fp16),
            engine._ptr(y), stream)

    def run(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            engine._check(lib.ct3_linear_prec(*args), "ct3_linear_prec")
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    run(3)                                            # module load, function attributes, L2 warm
    n = max(10, int(seconds * 1e3 / run(5)) + 1)
    return run(n), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="minimum timed time per shape")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_shapes.py times the GPU kernels; it needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card(0)}; library: {engine.LIB_PATH}")
    print(f"{'layers':28s} {'M':>7s} {'N':>5s} {'K':>5s} {'ms':>9s} {'TFLOP/s':>8s} {'launches':>8s} {'/iter':>5s}")
    step_ms = 0.0
    for name, M, Nout, K, act, products, fp16, per_iter in SHAPES:
        ms, n = time_shape(M, Nout, K, act, products, fp16, args.seconds, dev)
        tflops = 2.0 * M * Nout * K / (ms / 1e3) / 1e12
        step_ms += ITERS * per_iter * ms
        print(f"{name:28s} {M:7d} {Nout:5d} {K:5d} {ms:9.4f} {tflops:8.1f} {n:8d} {per_iter:5d}", flush=True)
        torch.cuda.empty_cache()
    print(f"GEMM ms per step from these shapes ({ITERS} iterations, fp16-plane corr_mlp.fc1): {step_ms:.1f}")


if __name__ == "__main__":
    main()
