"""Device timing of the resampling layer (engine.Resampler, Separator(..., sample_rate=)): development aid, not the bench.

- The two passes alone, for 180 s of 6-channel audio and 4 sources at 48, 96 and 192 kHz: the 6 audio planes to
  44.1 kHz, and the 24 stem planes back, trimmed to the input's length.  Bytes read and written and fp64 FMAs are
  computed from the shapes (one read of each input sample and one write of each output, ceil(K/up) FMAs per output);
  the share of the data sheet's 3.35 TB/s and the fp64 floor at 64 FMA/clk/SM and the card's max SM clock are beside.
- separate_channels of 180 s at C = 6 at 48 kHz against the same duration at 44.1 kHz (N = 1024), and the mono DSD100
  call at N = 2048 likewise.
Every pair is alternated, >= 10 timed calls each with CUDA events, medians and ranges.  It reads the card's name, power
limit and max SM clock in the same run.

    python tools/time_resample.py [--reps 10] [--seconds 180] [--out results.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Resampler, Separator  # noqa: E402
from time_channels import synth_params, card, timed  # noqa: E402

HBM_TBS = 3.35


def pass_cost(P, L_in, n_out, up, down):
    K = 20 * max(up, down) + 1
    Q = -(-K // up)
    return {"planes": P, "read_MB": P * L_in * 4e-6, "written_MB": P * n_out * 4e-6, "fp64_GFMA": P * n_out * Q * 1e-9,
            "taps_per_phase": Q}


def floors(cost, sms, sm_mhz):
    hbm = (cost["read_MB"] + cost["written_MB"]) * 1e6 / (HBM_TBS * 1e12) * 1e3
    fp64 = cost["fp64_GFMA"] * 1e9 / (64 * sms * sm_mhz * 1e6) * 1e3 if sm_mhz else None
    return hbm, fp64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_resample.py measures on the GPU and found none")
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "passes": [], "calls": []}
    print(json.dumps(res["card"]), flush=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sm_mhz = float(res["card"]["sm_max_mhz"]) if res["card"]["sm_max_mhz"] else None
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    sep = Separator(synth_params(513), frame_size=1024, hop=512, window="hanning", overlap=25)
    for rate in (48000, 96000, 192000):
        L = int(args.seconds * rate)
        down, back = Resampler(sep.ctx, rate, 44100), Resampler(sep.ctx, 44100, rate)
        x = torch.tensor(rng.uniform(-0.5, 0.5, (6, L)).astype(np.float32), device=dev)
        L44 = down.length(L)
        x44 = torch.empty((6, L44), device=dev)
        s44 = torch.tensor(rng.uniform(-0.5, 0.5, (24, L44)).astype(np.float32), device=dev)
        s = torch.empty((24, L), device=dev)
        ms = timed({"in": lambda: down.resample(x, out=x44), "back": lambda: back.resample(s44, num_out=L, out=s)}, args.reps)
        cfg = {"rate": rate, "ms": ms}
        for k, cost in (("in", pass_cost(6, L, L44, down.up, down.down)), ("back", pass_cost(24, L44, L, back.up, back.down))):
            hbm, fp64 = floors(cost, sms, sm_mhz)
            cost.update({"hbm_floor_ms": hbm, "fp64_floor_ms": fp64, "hbm_share": hbm / ms[k]["median"],
                         "fp64_share": fp64 / ms[k]["median"] if fp64 else None})
            cfg[k] = cost
        res["passes"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del x, x44, s44, s
    for name, N, nch in (("channels_C6", 1024, 6), ("mono_dsd", 2048, 1)):
        sp = sep if N == 1024 else Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25)
        planes = {}
        for rate in (44100, 48000):
            L = int(args.seconds * rate)
            t = np.arange(L) / rate
            cols = [0.2 * np.sin(2 * np.pi * 220 * (c + 1) * t) + 0.1 * rng.standard_normal(L) for c in range(nch)]
            planes[rate] = torch.tensor(np.stack(cols).astype(np.float32), device=dev)
        if nch == 1:
            runs = {"44100": lambda: sp.separate_device(planes[44100][0]),
                    "48000": lambda: sp.separate(planes[48000][0], sample_rate=48000)}
        else:
            runs = {"44100": lambda: sp.separate_channels(planes[44100]),
                    "48000": lambda: sp.separate_channels(planes[48000], sample_rate=48000)}
        cfg = {"call": name, "N": N, "channels": nch, "ms": timed(runs, args.reps)}
        cfg["ratio_48000_over_44100"] = cfg["ms"]["48000"]["median"] / cfg["ms"]["44100"]["median"]
        res["calls"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del planes
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
