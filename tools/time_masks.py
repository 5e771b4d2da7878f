"""Device timing of the masks output (dcs_separate_masks) against the stems call (dcs_separate_audio) of the DSD100
network (development aid, not the bench).

One seeded 180 s clip at N = 2048: warm-up, then the masks call and the stems call alternated, each timed whole with
CUDA events and per stage with dcs_profile (its CUDA events); medians over --reps calls of each, with the card's name,
power limit and maximum SM clock read in the same run, the launch counts and the workspace each mode holds.

    python tools/time_masks.py [--reps 15] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Separator  # noqa: E402

SR = 44100


def synth_params(F, seed=0):
    """DSD100 parameter list with Glorot-uniform weights (the shapes of tools/quick_time.py)"""
    rng = np.random.default_rng(seed)
    shapes = [(50, 1, 1, F), (50,), (50,), (50, 50, 15, 1), (50,), (50,), (800, 128), (128,), (128, 800), (800,),
              (128, 800), (800,), (128, 800), (800,), (4,)]
    out = []
    for s in shapes:
        if len(s) == 4:
            a = np.sqrt(6.0 / ((s[0] + s[1]) * s[2] * s[3]))
        elif len(s) == 2:
            a = np.sqrt(6.0 / (s[0] + s[1]))
        else:
            a = 0.1
        out.append(rng.uniform(-a, a, size=s).astype(np.float32))
    return out


def clip(seconds, seed=1234):
    rng = np.random.default_rng(seed)
    L = int(seconds * SR)
    t = np.arange(L) / SR
    x = 0.2 * np.sin(2 * np.pi * 220 * t) + 0.1 * np.sin(2 * np.pi * 330 * t) + 0.1 * rng.standard_normal(L)
    return x.clip(-0.99, 0.99).astype(np.float32)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, sm_max = [v.strip() for v in q.split(",")]
    except Exception:  # noqa: BLE001
        power, sm_max = None, None
    return {"gpu": name, "power_limit_w": power, "sm_max_mhz": sm_max}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--N", type=int, default=2048)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "seconds": args.seconds, "N": args.N, "reps": args.reps}
    print(json.dumps(res["card"]), flush=True)
    N, dev = args.N, torch.device("cuda", 0)
    x = torch.tensor(clip(args.seconds), device=dev)
    L = x.numel()
    params = synth_params(N // 2 + 1)
    seps = {k: Separator(params, frame_size=N, hop=512, window="hanning", overlap=25) for k in ("masks", "stems")}
    T, ldf = seps["masks"].stft.num_frames(L), seps["masks"].stft.ldf
    outs = {"masks": torch.empty((4, T, ldf), dtype=torch.float32, device=dev),
            "stems": torch.empty((4, L), dtype=torch.float32, device=dev)}
    runs = {"masks": lambda: seps["masks"].separate_masks(x, out=outs["masks"]),
            "stems": lambda: seps["stems"].separate_device(x, outs["stems"])}
    for _ in range(3):
        for f in runs.values():
            f()
    torch.cuda.synchronize()
    total = {k: [] for k in runs}
    stages = {k: {} for k in runs}
    launches = {}
    for _ in range(args.reps):
        for k, f in runs.items():          # alternated: both modes see the same state of the shared machine
            sep = seps[k]
            sep.ctx.profile(False)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = sep.ctx.launch_count()
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            launches[k] = sep.ctx.launch_count() - n0
            total[k].append(e0.elapsed_time(e1))
            sep.ctx.profile(True)          # a separate call for the stage breakdown: the events add a little time
            f()
            torch.cuda.synchronize()
            per = {}
            for name, ms in sep.ctx.profile_read():
                per[name] = per.get(name, 0.0) + ms
            sep.ctx.profile(False)
            for name, ms in per.items():
                stages[k].setdefault(name, []).append(ms)
    res["frames"], res["ldf"], res["launches"] = T, ldf, launches
    res["call_ms_median"] = {k: float(np.median(v)) for k, v in total.items()}
    res["call_ms_min"] = {k: float(np.min(v)) for k, v in total.items()}
    res["stage_ms_median"] = {k: {n: float(np.median(v)) for n, v in s.items()} for k, s in stages.items()}
    res["workspace_bytes"] = {k: seps[k].ctx.workspace_bytes() for k in seps}
    a = res["stage_ms_median"]["masks"].get("dec_convT1_mask_xfade")
    b = res["stage_ms_median"]["stems"].get("dec_convT1_mask_xfade")
    res["mask_stage_masks_over_stems"] = a / b if a and b else None
    # compulsory bytes of the mask stage: Ŝ mode reads X (8 B) and writes 4 spectra (32 B) per (t, f); masks mode
    # writes 4 masks (16 B); both read the decoder activations G
    F = N // 2 + 1
    res["mask_stage_bytes_GB"] = {"stems": T * F * 40 / 1e9, "masks": T * F * 16 / 1e9}
    print(json.dumps(res, indent=1), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
