"""Host-to-host throughput of one long multichannel recording (development aid, not the bench):
Separator.separate_long_channels against the same recording cut by the caller into 120 s clips through
separate_channels_batch, and a 16-channel recording the whole-recording batch cannot hold.

  (a) 30 min of 6-channel int16 at 48 kHz, N = 2048 (the DSD100-shaped synthetic params of tools/time_channels.py),
      without the filter and with K = 2, W = 2: the long call (120 s segments) and the caller's 120 s cuts through
      separate_channels_batch in one call (which leaves seams at every cut), alternated after a warm-up;
  (b) 30 min of 16-channel int16 at 44.1 kHz, no filter: the long call.
The signal is 60 s of time_channels.clip tiled to length, in pinned host memory, stems into pinned buffers.  Host wall
clock around each call, ending in a device synchronise, as audio-seconds per second (median and range of --reps).
Beside them: the bytes each call moves over the host link (from the shapes) and the least time the link takes for them
at the pinned H2D / D2H rates measured in the same run (the two directions overlap), the kernel time of one long call
summed over the pipeline's outermost dcs_profile scopes, and the ctx's workspace after the call.  It reads the card's
name, power limit and max SM clock in the same run, and exits without a GPU.

    python tools/time_long_channels.py [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Separator  # noqa: E402
from time_channels import card, clip, synth_params  # noqa: E402

MODEL = 44100
NSRC = 4
SEG = 120.0


def pinned(shape, dtype):
    return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True).numpy()


def recording(seconds, rate, nch, seed=2026):
    """int16 [seconds * rate, nch], pinned: 60 s of time_channels.clip at 0.8 of full scale, tiled"""
    base = np.round(clip(60.0 * rate / MODEL, nch, seed=seed).T * 0.8 * 32767).astype(np.int16)
    L = int(seconds * rate)
    p = pinned((L, nch), np.int16)
    for k in range(0, L, base.shape[0]):
        n = min(base.shape[0], L - k)
        p[k:k + n] = base[:n]
    return p


def wall(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def rates(v, audio_s):
    r = [audio_s / t for t in v]
    return {"audio_s_per_s_median": float(np.median(r)), "min": float(np.min(r)), "max": float(np.max(r)),
            "wall_s": [float(t) for t in v]}


def link_rates(nbytes=1 << 30):
    """pinned host <-> device copy rates in bytes/s, CUDA events, median of 5"""
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {}
    for name, f in (("h2d", lambda: d.copy_(h, non_blocking=True)), ("d2h", lambda: h.copy_(d, non_blocking=True))):
        ts = []
        for _ in range(5):
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        out[name] = nbytes / float(np.median(ts))
    return out


# the pipeline's outermost dcs_profile scopes (api.cu batch_pipeline, resample.cu): the others nest inside them
TOP_SCOPES = ("pcm16_decode_separate", "pcm16_encode", "pcm16_separate", "resample_decode", "resample_decode_downmix",
              "resample_encode")


def kernel_ms(sep, call):
    """device ms of one call: the sum of its outermost profile scopes (the copies run on their own streams)"""
    sep.ctx.profile(True)
    call()
    torch.cuda.synchronize()
    rec = sep.ctx.profile_read()
    sep.ctx.profile(False)
    return float(sum(ms for n, ms in rec if n in TOP_SCOPES))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--minutes", type=float, default=30.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_long_channels: no CUDA device")
    res = {"card": card(), "segment_seconds": SEG, "minutes": a.minutes}
    link = link_rates()
    res["link_bytes_per_s"] = link
    sep = Separator(synth_params(1025), frame_size=2048, hop=512, window="hanning", overlap=25)
    seconds = a.minutes * 60.0

    # (a) 6 channels at 48 kHz: the long call against the caller's 120 s cuts
    rate, nch = 48000, 6
    rec = recording(seconds, rate, nch)
    L = rec.shape[0]
    out = pinned((NSRC, L, nch), np.int16)
    cut = int(SEG * rate)
    clips = [rec[k:k + cut] for k in range(0, L, cut)]
    outs = [pinned((NSRC, c.shape[0], nch), np.int16) for c in clips]
    moved = rec.nbytes + out.nbytes
    for wiener, radius in ((0, 0), (2, 2)):
        key = "6ch_48k_wiener%d" % wiener
        long_call = lambda: sep.separate_long_channels(rec, out=out, wiener=wiener, wiener_radius=radius,  # noqa: E731
                                                       sample_rate=rate, segment_seconds=SEG)
        cut_call = lambda: sep.separate_channels_batch(clips, outs=outs, wiener=wiener, wiener_radius=radius,  # noqa: E731
                                                       sample_rate=rate)
        long_call()
        cut_call()
        t_long, t_cut = [], []
        for _ in range(a.reps):
            t_long.append(wall(long_call))
            t_cut.append(wall(cut_call))
        segs = sep.long_segments(L, wiener, radius, rate, SEG)
        fresh = Separator(synth_params(1025), frame_size=2048, hop=512, window="hanning", overlap=25)
        fresh.separate_long_channels(rec, out=out, wiener=wiener, wiener_radius=radius, sample_rate=rate, segment_seconds=SEG)
        res[key] = {"long": rates(t_long, seconds), "caller_cuts_120s": rates(t_cut, seconds), "segments": len(segs),
                    "model_samples_per_core": float(sum(s.model_stop - s.model_start for s in segs)) / sum(
                        s.out_stop - s.out_start for s in segs) * rate / MODEL,
                    "kernel_ms_long": kernel_ms(sep, long_call), "bytes_over_link": moved,
                    "link_bound_s": max(rec.nbytes / link["h2d"], out.nbytes / link["d2h"]),
                    "workspace_bytes_long": fresh.ctx.workspace_bytes()}
        fresh2 = Separator(synth_params(1025), frame_size=2048, hop=512, window="hanning", overlap=25)
        fresh2.separate_channels_batch(clips, outs=outs, wiener=wiener, wiener_radius=radius, sample_rate=rate)
        res[key]["workspace_bytes_caller_cuts"] = fresh2.ctx.workspace_bytes()
        del fresh, fresh2
        print(json.dumps({key: res[key]}), flush=True)
    del rec, out, clips, outs
    if hasattr(torch._C, "_host_emptyCache"):
        torch._C._host_emptyCache()

    # (b) 16 channels at 44.1 kHz: the long call only
    rate, nch = MODEL, 16
    rec = recording(seconds, rate, nch)
    L = rec.shape[0]
    out = pinned((NSRC, L, nch), np.int16)
    long_call = lambda: sep.separate_long_channels(rec, out=out, segment_seconds=SEG)  # noqa: E731
    long_call()
    t_long = [wall(long_call) for _ in range(a.reps)]
    fresh = Separator(synth_params(1025), frame_size=2048, hop=512, window="hanning", overlap=25)
    fresh.separate_long_channels(rec, out=out, segment_seconds=SEG)
    res["16ch_441k"] = {"long": rates(t_long, seconds), "segments": len(sep.long_segments(L, segment_seconds=SEG)),
                        "kernel_ms_long": kernel_ms(sep, long_call), "bytes_over_link": rec.nbytes + out.nbytes,
                        "link_bound_s": max(rec.nbytes / link["h2d"], out.nbytes / link["d2h"]),
                        "workspace_bytes_long": fresh.ctx.workspace_bytes()}
    print(json.dumps({"16ch_441k": res["16ch_441k"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
