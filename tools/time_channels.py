"""Device timing of C-channel stems (Separator.separate_channels: the downmix's masks applied inside the inverse STFT)
against the keep-channels mode and the mono call (development aid, not the bench).  Keep-channels without the Wiener
post-filter takes the C = 2 path; timing it next to separate_channels at C = 2 shows what its entry point adds.

One seeded 180 s clip at N = 2048 and N = 1024: warm-up, then separate_keep_channels and separate_channels at C = 2
alternated, then separate and separate_channels at C = 1 alternated, then separate_channels at C = 6 on its own, >= 10
timed calls each with CUDA events (medians and ranges); the dcs_profile stage table of one call of each, next to the
bytes the mask stage and the inverse STFT must move, computed from the buffer shapes; the workspace each call leaves.
It reads the card's name, power limit and max SM clock in the same run.

    python tools/time_channels.py [--reps 12] [--out results.json]
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


def stereo_clip(seconds, seed=1234):
    rng = np.random.default_rng(seed)
    L = int(seconds * SR)
    t = np.arange(L) / SR
    common = 0.2 * np.sin(2 * np.pi * 220 * t) + 0.1 * rng.standard_normal(L)
    left = common + 0.1 * np.sin(2 * np.pi * 330 * t) + 0.05 * rng.standard_normal(L)
    right = 0.8 * common + 0.1 * np.sin(2 * np.pi * 550 * t) + 0.05 * rng.standard_normal(L)
    return np.stack([left, right], axis=1).clip(-0.99, 0.99).astype(np.float32)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, sm_max = [v.strip() for v in q.split(",")]
    except Exception:  # noqa: BLE001
        power, sm_max = None, None
    return {"gpu": name, "power_limit_w": power, "sm_max_mhz": sm_max}


def stages(sep, call):
    sep.ctx.profile(True)
    call()
    torch.cuda.synchronize()
    rec = sep.ctx.profile_read()
    sep.ctx.profile(False)
    out = {}
    for name, ms in rec:
        out[name] = out.get(name, 0.0) + ms
    return out


def clip(seconds, nch, seed=1234):
    """nch channels: two shared components at per-channel gains and delays, plus a little independent noise"""
    rng = np.random.default_rng(seed)
    L = int(seconds * SR)
    t = np.arange(L) / SR
    a = 0.2 * np.sin(2 * np.pi * 220 * t) + 0.1 * rng.standard_normal(L)
    b = 0.1 * np.sin(2 * np.pi * 330 * t) + 0.1 * rng.standard_normal(L)
    cols = [g * np.roll(a, d) + h * np.roll(b, e) + 0.02 * rng.standard_normal(L)
            for g, h, d, e in zip(rng.uniform(0.3, 1, nch), rng.uniform(-1, 1, nch), rng.integers(0, 40, nch), rng.integers(0, 40, nch))]
    return np.stack(cols).clip(-0.99, 0.99).astype(np.float32)          # planes [C, L]


def shape_bytes(N, L, nch, nsrc=4, hop=512):
    """MB the mask stage writes and the inverse STFT reads at the least (every plane once), and the spectra held"""
    plane = ((L + hop - 1) // hop + 2) * ((N // 2 + 1 + 7) // 8 * 8)
    mb = 1e-6
    return {"mask_stage_writes_M": nsrc * plane * 4 * mb, "mask_stage_reads_X": 0.0,
            "istft_reads_X_once": nch * plane * 8 * mb, "istft_reads_M_once": nsrc * plane * 4 * mb,
            "istft_reads_no_reuse": nsrc * nch * plane * 12 * mb, "spectra_held": (plane * 8 + nsrc * plane * 4) * mb}


def timed(runs, reps):
    """the calls of `runs` alternated, reps timed rounds after three warm-up rounds -> ms per call"""
    for _ in range(3):
        for f in runs.values():
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    for _ in range(reps):
        for k, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    return {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_channels.py measures on the GPU and found none")
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "configs": []}
    print(json.dumps(res["card"]), flush=True)
    dev = torch.device("cuda", 0)
    x6 = torch.tensor(clip(args.seconds, 6), device=dev)
    x2, x1 = x6[:2].contiguous(), x6[:1].contiguous()
    L = x6.shape[1]
    for N in (2048, 1024):
        params = synth_params(N // 2 + 1)

        def make():
            return Separator(params, frame_size=N, hop=512, window="hanning", overlap=25)
        keep, chan, mono = make(), make(), make()          # a context each: the workspace figures are each call's own
        o8, o4, o24 = (torch.empty((n, L), dtype=torch.float32, device=dev) for n in (8, 4, 24))
        calls = {"keep_channels_C2": (keep, lambda: keep.separate_keep_channels(x2, o8)),
                 "channels_C2": (chan, lambda: chan.separate_channels(x2, o8)),
                 "mono": (mono, lambda: mono.separate_device(x1[0], o4)),
                 "channels_C1": (chan, lambda: chan.separate_channels(x1, o4)),
                 "channels_C6": (chan, lambda: chan.separate_channels(x6, o24))}
        ms = {}
        for group in (("keep_channels_C2", "channels_C2"), ("mono", "channels_C1"), ("channels_C6",)):
            ms.update(timed({k: calls[k][1] for k in group}, args.reps))
        launches = {}
        for k, (s, f) in calls.items():
            n0 = s.ctx.launch_count()
            f()
            launches[k] = s.ctx.launch_count() - n0
        torch.cuda.synchronize()
        cfg = {"N": N, "ms": ms, "launches": launches, "stages_ms": {k: stages(s, f) for k, (s, f) in calls.items()},
               "workspace_MB": {"keep_channels": keep.ctx.workspace_bytes() / 1e6, "channels": chan.ctx.workspace_bytes() / 1e6,
                                "mono": mono.ctx.workspace_bytes() / 1e6},
               "shape_MB": {"C2": shape_bytes(N, L, 2), "C6": shape_bytes(N, L, 6)}}
        res["configs"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del keep, chan, mono
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
