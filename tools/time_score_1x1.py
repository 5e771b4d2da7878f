"""Per-stage device time of the score-informed build_ca_1x1 network (dcs_profile) on a 30 s clip at the trainer's
geometry (N = 4096, hop 512, F = 2049, tc 30, overlap 25), with the algorithmic FLOPs of each stage, and the
17-array build_ca score net timed in the same run for context.  Synthetic weights (timing does not depend on them).

    python tools/time_score_1x1.py [--seconds 30] [--reps 5] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

from deepconvsep_b200.engine import Separator  # noqa: E402
from oracle import nets, pipeline  # noqa: E402
import score1x1_oracle as s1  # noqa: E402  (synthetic weights and layer widths)


def flops_1x1(T, P, F=2049, tc=30):
    """algorithmic FLOPs (2 per MAC) per stage; the decoder counts every tap, the K clipping skips only zeros"""
    W = [F] + s1.widths_1x1(F)
    C = [4, 30, 50, 70, 100, 200, 200]
    kh = [0, 1, 1, 1, 1, 10, 10]
    Tp = max(T, (P - 1) * 5 + tc)
    rows = [0, Tp, Tp, Tp, Tp, Tp - 9, Tp - 18]
    h = [0, tc, tc, tc, tc, tc - 9, tc - 18]
    f = {}
    for l in range(1, 7):
        f["enc_conv%d_gemm" % l] = 2.0 * rows[l] * W[l] * C[l] * C[l - 1] * kh[l] * 5
        if l >= 2:   # InverseLayer(conv l): every output of conv l feeds kh*5 inputs
            f["dec_convT%d_gemm" % l] = 2.0 * P * h[l] * W[l] * C[l] * C[l - 1] * kh[l] * 5
    f["conv1x1_gemm"] = 2.0 * P * h[6] * W[6] * 200 * 200
    f["dec_convT1_mask_xfade"] = 2.0 * P * tc * W[1] * 30 * 4 * 5
    return f


def run(sep, mix, filters, reps):
    lib, h = sep.lib, sep.ctx.handle
    sep.separate_score(mix, filters)                   # warm-up: workspace, weights in L2, clocks
    torch.cuda.synchronize()
    tot = {}
    wall = []
    for _ in range(reps):
        lib.dcs_profile(h, 1)
        sep.separate_score(mix, filters)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 16)
        ms = np.zeros(4096, dtype=np.float32)
        n = lib.dcs_profile_read(h, buf, len(buf), ms.ctypes.data, ms.size)
        lib.dcs_profile(h, 0)
        names = buf.value.decode().split("\n")[:n]
        per = {}
        for nm, t in zip(names, ms[:n]):
            per[nm] = per.get(nm, 0.0) + float(t)
        for k, v in per.items():
            tot.setdefault(k, []).append(v)
        wall.append(sum(per.values()))
    return {k: float(np.median(v)) for k, v in tot.items()}, float(np.median(wall)), names.count("dec_convT1_mask_xfade")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    mix, _ = pipeline.synth_mixture(args.seconds, 12)
    N, hop, F = 4096, 512, 2049
    T = int(np.ceil(mix.size / hop)) + 2
    rng = np.random.default_rng(1)
    raw = np.full((4, T, F), 1e-18, dtype=np.float32)
    for j in range(4):
        for _ in range(T // 20):
            t0, b0 = rng.integers(0, T - 40), rng.integers(1, F - 40)
            raw[j, t0:t0 + 40, b0:b0 + 30] = 1.0
    filters = (raw / raw.sum(axis=0)).astype(np.float32)
    out = {"device": dev, "power_limit": power, "seconds": args.seconds, "N": N, "hop": hop, "frames": T}
    sep = Separator(s1.make_synthetic_params_1x1(seed=1), arch="bach10_score_1x1", frame_size=N, hop=hop,
                    window="blackmanharris", overlap=25, patcher="util", scale_factor=0.2, feat_size=F, time_context=30)
    P = sep.num_patches(T)
    stages, total, chunks = run(sep, mix, filters, args.reps)
    fl = flops_1x1(T, P)
    out["score_1x1"] = {"patches": P, "chunks": chunks, "total_ms": total, "workspace_bytes": int(sep.lib.dcs_workspace_bytes(sep.ctx.handle)),
                        "stages": {k: {"ms": v, "gflop": fl.get(k, 0.0) / 1e9,
                                       "tflops": fl.get(k, 0.0) / (v * 1e-3) / 1e12 if k in fl and v > 0 else None}
                                   for k, v in sorted(stages.items(), key=lambda kv: -kv[1])},
                        "gflop_total": sum(fl.values()) / 1e9}
    del sep
    torch.cuda.empty_cache()
    sep = Separator(nets.make_synthetic_params("bach10_score", F, seed=1), arch="bach10_score", frame_size=N, hop=hop,
                    window="blackmanharris", overlap=25, patcher="util", scale_factor=0.2, feat_size=F)
    stages, total, _ = run(sep, mix, filters, args.reps)
    out["score_build_ca"] = {"total_ms": total, "stages": stages}
    print("%s, power limit %s; %.0f s clip, N=%d hop %d: %d frames, %d patches, %d decoder chunks"
          % (dev, power, args.seconds, N, hop, T, P, out["score_1x1"]["chunks"]))
    print("%-24s %10s %10s %8s" % ("build_ca_1x1 stage", "ms", "GFLOP", "TFLOP/s"))
    for k, v in out["score_1x1"]["stages"].items():
        print("%-24s %10.3f %10.1f %8s" % (k, v["ms"], v["gflop"], "%.1f" % v["tflops"] if v["tflops"] else "-"))
    print("%-24s %10.3f %10.1f" % ("total", out["score_1x1"]["total_ms"], out["score_1x1"]["gflop_total"]))
    print("build_ca score net, same clip: %.3f ms" % out["score_build_ca"]["total_ms"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
