"""Device timing of the multichannel Wiener post-filter on keep-channels stems (development aid, not the bench).

One seeded 180 s stereo clip through the DSD100 network in keep-channels mode at N = 2048: warm-up, then
K = 0, 1, 2, 3 EM iterations at covariance radius W = 0 (the whole clip) and K = 1, 2, 3 at each --radii W (sliding
window of W chunks to either side), alternated, >= 12 timed calls each with CUDA events; the dcs_profile stage
breakdown of one call per (K, W); and each Wiener stage's achieved bandwidth against the bytes it must move, computed
from the shapes.  Then the device workspace (dcs_workspace_bytes) of a --long-seconds recording separated whole and of
the longest of --parts segments (deepconvsep_b200.longclip, K = 2, W = 2), each on a fresh context.
The card's name, power limit and SM clock are read in the same run.

    python tools/time_wiener.py [--reps 12] [--seconds 180] [--radii 1,4] [--long-seconds 1800] [--parts 4] [--out results.json]
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

from deepconvsep_b200 import longclip  # noqa: E402
from deepconvsep_b200.engine import Separator  # noqa: E402
from time_channels import synth_params, stereo_clip, stages  # noqa: E402

NSRC, CHUNK = 4, 128      # sources; frames per partial-sum chunk (csrc/wiener.cu kWienerFrames)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    return {"gpu": name, "torch_name": torch.cuda.get_device_name(0), "power_limit_w": power, "sm_clock_mhz": sm,
            "sm_max_mhz": sm_max}


def wiener_bytes(T, F, nsrc=NSRC, radius=0):
    """bytes each stage must move: the init pass reads the float masks and X and writes the stems; an EM pass reads
    the stems and X and writes the stems;
    every pass but the last EM one writes per-chunk partial sums that its reduce reads back -- with a radius W >= 1
    each chunk reads the partials of its (up to 2W + 1) window chunks and writes its own R"""
    n = -(-T // CHUNK)
    plane = T * F * 8
    partials = n * nsrc * 4 * F * 8
    reread = partials if radius == 0 else sum(min(n - 1, c + radius) - max(0, c - radius) + 1 for c in range(n)) * partials // n
    write_q = 0 if radius == 0 else partials
    init = (nsrc // 2 + 2 + 2 * nsrc) * plane + partials + reread + write_q
    em = (4 * nsrc + 2) * plane
    return {"plane_MB": plane / 1e6, "partials_MB": partials / 1e6, "reduce_read_MB": reread / 1e6,
            "init_GB": init / 1e9, "em_last_GB": em / 1e9, "em_GB": (em + partials + reread + write_q) / 1e9}


def workspace(params, N, audio, wiener, radius):
    """dcs_workspace_bytes of a fresh context after separating `audio` in keep-channels mode"""
    sep = Separator(params, frame_size=N, hop=512, window="hanning", overlap=25)
    x = torch.tensor(np.ascontiguousarray(audio.T), device=torch.device("cuda", 0))
    sep.separate_keep_channels(x, wiener=wiener, wiener_radius=radius)
    torch.cuda.synchronize()
    b = sep.ctx.workspace_bytes()
    del sep, x
    torch.cuda.empty_cache()
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--radii", default="1,4")
    ap.add_argument("--long-seconds", type=float, default=1800.0)
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    radii = [int(r) for r in args.radii.split(",") if r]
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
    Ks = [(K, 0) for K in (0, 1, 2, 3)] + [(K, W) for W in radii for K in (1, 2, 3)]
    runs = {K: (lambda K=K: sep.separate_keep_channels(x2, out, wiener=K[0], wiener_radius=K[1])) for K in Ks}
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
    name = lambda k: "K%d_W%d" % k  # noqa: E731
    res.update(frames=T, bins=F, bytes={"W%d" % W: wiener_bytes(T, F, radius=W) for W in [0] + radii},
               stages_ms={name(k): v for k, v in prof.items()},
               ms={name(K): {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                   for K, v in ms.items()})
    bw = {}
    for K, W in Ks:
        if K == 0:
            continue
        p, b = prof[(K, W)], wiener_bytes(T, F, radius=W)
        em_bytes = (K - 1) * b["em_GB"] + b["em_last_GB"]
        bw[name((K, W))] = {"wiener_init_ms": p.get("wiener_init"), "wiener_em_ms": p.get("wiener_em"),
                            "wiener_init_GBps": b["init_GB"] / (p["wiener_init"] / 1e3),
                            "wiener_em_GBps": em_bytes / (p["wiener_em"] / 1e3),
                            "clip_ms_over_K0": float(np.median(ms[(K, W)]) - np.median(ms[(0, 0)]))}
    res["wiener_bandwidth"] = bw
    del sep, x2, out
    torch.cuda.empty_cache()
    # workspace of a long recording: whole versus the longest segment when cut into --parts (K = 2, W = 2)
    params = synth_params(N // 2 + 1)
    long_audio = stereo_clip(args.long_seconds)
    segs = longclip.plan_segments(long_audio.shape[0], args.parts, N, 512, 30, 25, wiener_reach=2 * 2)
    longest = max(segs, key=lambda s: s.in_stop - s.in_start)
    res["workspace"] = {"seconds": args.long_seconds, "parts": len(segs),
                        "longest_segment_s": (longest.in_stop - longest.in_start) / 44100.0,
                        "whole_K2_W0_bytes": workspace(params, N, long_audio, 2, 0),
                        "whole_K2_W2_bytes": workspace(params, N, long_audio, 2, 2),
                        "segment_K2_W2_bytes": workspace(params, N, long_audio[longest.in_start:longest.in_stop], 2, 2)}
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
