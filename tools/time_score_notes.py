"""Per-clip cost of the two ways to feed the score-informed nets, at the trainer's geometry (N = 4096, hop 512,
F = 2049, overlap 25, util patcher), for build_ca (17 arrays) and build_ca_1x1 (22 arrays):

  (a) filters: score.score_filters on the host (expandMidi + filterSpec, four dense planes) + Separator.separate_score
      (the planes are copied to the device and multiplied by the magnitude there);
  (b) notes:   score.score_melody on the host (expandMidi only) + Separator.separate_notes (the note table is
      rasterised on the device straight into the network's input channels).

For each: the host time of the score prelude, the device time of the separation call (CUDA events on the stream,
host audio in, host stems out), the `score_channels` stage of dcs_profile, and a check that both paths give the same
bits.  Synthetic Bach10-like scores (about 7 notes/s over 4 instruments) and synthetic weights.

    python tools/time_score_notes.py [--seconds 30 180] [--reps 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

from deepconvsep_b200 import score  # noqa: E402
from deepconvsep_b200.engine import Separator  # noqa: E402
from oracle import nets, pipeline  # noqa: E402
import score1x1_oracle as s1  # noqa: E402  (synthetic weights of the 1x1 net)

INSTS = ["bassoon_b", "clarinet_b", "saxophone_b", "violin_b"]
RANGES = {"bassoon_b": (2, 3), "clarinet_b": (4, 5), "saxophone_b": (3, 4), "violin_b": (4, 6)}   # octaves


def write_scores(d, seconds, seed):
    """one `onset,offset,note` line per note, notes of 0.3-0.9 s back to back with occasional short rests"""
    rng = np.random.default_rng(seed)
    names = ["C", "D", "E", "F", "G", "A", "B", "Bb", "F#", "Eb"]
    nnotes = 0
    for k in INSTS:
        t, lines = 0.05, []
        lo, hi = RANGES[k]
        while t < seconds:
            d0 = rng.uniform(0.3, 0.9)
            lines.append("%.2f,%.2f,%s%d" % (t, min(t + d0, seconds), names[rng.integers(len(names))], rng.integers(lo, hi + 1)))
            t += d0 + (rng.uniform(0.05, 0.15) if rng.random() < 0.3 else 0.0)
        open(os.path.join(d, k + ".txt"), "w").write("\n".join(lines) + "\n")
        nnotes += len(lines)
    return nnotes


def profile_stage(sep, name):
    return sum(ms for nm, ms in sep.ctx.profile_read() if nm == name)


def time_path(sep, mix, prelude, call, reps):
    """median host ms of the prelude, device ms of the call (events), score_channels ms; the last outputs"""
    host, dev, stage = [], [], []
    for i in range(reps + 1):                         # the first run warms up workspace, weights and clocks
        t0 = time.perf_counter()
        arg = prelude()
        t1 = time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sep.ctx.profile(True)
        e0.record()
        out = call(arg)
        e1.record()
        torch.cuda.synchronize()
        st = profile_stage(sep, "score_channels")
        sep.ctx.profile(False)
        if i:
            host.append((t1 - t0) * 1e3)
            dev.append(e0.elapsed_time(e1))
            stage.append(st)
    return dict(host_ms=float(np.median(host)), device_ms=float(np.median(dev)), score_channels_ms=float(np.median(stage))), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, nargs="+", default=[30.0, 180.0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.cuda.get_device_name(0)
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = "unknown"
    N, hop, F = 4096, 512, 2049
    nets_ = {"build_ca (17 arrays)": nets.make_synthetic_params("bach10_score", F, seed=1),
             "build_ca_1x1 (22 arrays)": s1.make_synthetic_params_1x1(seed=1)}
    out = {"device": dev, "power_limit,clocks.max.sm,clocks.sm": smi, "N": N, "hop": hop, "rows": []}
    print("%s; power limit, max SM clock, SM clock: %s" % (dev, smi))
    print("%-26s %6s %6s %6s  %-8s %10s %10s %16s %10s" % ("network", "clip_s", "frames", "notes", "path", "host_ms",
                                                          "device_ms", "score_channels_ms", "same_bits"))
    for name, params in nets_.items():
        sep = Separator(params, frame_size=N, hop=hop, window="blackmanharris", overlap=25, patcher="util", scale_factor=0.2,
                        feat_size=F)
        for seconds in args.seconds:
            mix, _ = pipeline.synth_mixture(seconds, 12)
            T = int(np.ceil(mix.size / hop)) + 2
            with tempfile.TemporaryDirectory() as d:
                nnotes = write_scores(d, seconds, 3)
                kw = dict(frameSize=N, hopSize=hop, duration=seconds)
                a, ya = time_path(sep, mix, lambda: score.score_filters(d, INSTS, T, F, **kw),
                                  lambda f: sep.separate_score(mix, f), args.reps)
                b, yb = time_path(sep, mix, lambda: score.score_melody(d, INSTS, T, **kw),
                                  lambda m: sep.separate_notes(mix, m), args.reps)
            same = ya.tobytes() == yb.tobytes()
            for path, r in (("filters", a), ("notes", b)):
                print("%-26s %6.0f %6d %6d  %-8s %10.1f %10.2f %16.4f %10s" % (name, seconds, T, nnotes, path, r["host_ms"],
                                                                             r["device_ms"], r["score_channels_ms"], same))
                out["rows"].append(dict(r, network=name, seconds=seconds, frames=T, notes=nnotes, path=path, same_bits=same))
        del sep
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
