"""Device timing of the multichannel Wiener post-filter on keep-channels stems (development aid, not the bench).

One seeded 180 s stereo clip through the DSD100 network in keep-channels mode at N = 2048: warm-up, then
K = 0, 1, 2, 3 EM iterations alternated, >= 12 timed calls each with CUDA events; the dcs_profile stage breakdown of
one call per K; and each Wiener stage's achieved bandwidth against the bytes it must move, computed from the shapes.
The card's name, power limit and SM clock are read in the same run.

    python tools/time_wiener.py [--reps 12] [--seconds 180] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Separator  # noqa: E402
from time_keep_channels import synth_params, stereo_clip, stages  # noqa: E402

NSRC, CHUNK = 4, 128      # sources; frames per partial-sum chunk (csrc/wiener.cu kWienerFrames)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    return {"gpu": name, "torch_name": torch.cuda.get_device_name(0), "power_limit_w": power, "sm_clock_mhz": sm,
            "sm_max_mhz": sm_max}


def wiener_bytes(T, F, nsrc=NSRC):
    """bytes each stage must move: the init pass reads the stems and X; an EM pass reads them and writes the stems;
    every pass but the last EM one writes per-chunk partial sums that its reduce reads back"""
    plane = T * F * 8
    partials = -(-T // CHUNK) * nsrc * 4 * F * 8
    init = (2 * nsrc + 2) * plane + 2 * partials
    em = (4 * nsrc + 2) * plane
    return {"plane_MB": plane / 1e6, "partials_MB": partials / 1e6, "init_GB": init / 1e9, "em_last_GB": em / 1e9,
            "em_GB": (em + 2 * partials) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_wiener.py measures on the GPU; no CUDA device")
    N = 2048
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "N": N}
    print(json.dumps(res["card"]), flush=True)
    audio = stereo_clip(args.seconds)
    L = audio.shape[0]
    dev = torch.device("cuda", 0)
    x2 = torch.tensor(np.ascontiguousarray(audio.T), device=dev)
    sep = Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25)
    T, F = sep.stft.num_frames(L), N // 2 + 1
    out = torch.empty((8, L), dtype=torch.float32, device=dev)
    Ks = (0, 1, 2, 3)
    runs = {K: (lambda K=K: sep.separate_keep_channels(x2, out, wiener=K)) for K in Ks}
    for _ in range(3):
        for f in runs.values():
            f()
    torch.cuda.synchronize()
    ms = {K: [] for K in Ks}
    for _ in range(args.reps):
        for K, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ms[K].append(e0.elapsed_time(e1))
    prof = {K: stages(sep, f) for K, f in runs.items()}
    b = wiener_bytes(T, F)
    res.update(frames=T, bins=F, bytes=b, stages_ms={str(k): v for k, v in prof.items()},
               ms={str(K): {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                   for K, v in ms.items()})
    bw = {}
    for K in Ks[1:]:
        p = prof[K]
        em_bytes = (K - 1) * b["em_GB"] + b["em_last_GB"]
        bw[str(K)] = {"wiener_init_ms": p.get("wiener_init"), "wiener_em_ms": p.get("wiener_em"),
                      "wiener_init_GBps": b["init_GB"] / (p["wiener_init"] / 1e3),
                      "wiener_em_GBps": em_bytes / (p["wiener_em"] / 1e3),
                      "clip_ms_over_K0": float(np.median(ms[K]) - np.median(ms[0]))}
    res["wiener_bandwidth"] = bw
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
