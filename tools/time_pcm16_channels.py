"""Host-to-host throughput of 6-channel int16 wavs (development aid, not the bench): the float route the scripts take
today against the int16 multi-clip scheduler (Separator.separate_pcm16_channels_batch).

Twelve seeded 6-channel int16 clips of 60 to 180 s in pinned host memory, stems into pinned int16 buffers, the
DSD100-shaped synthetic params of tools/time_channels.py, at N = 2048 and N = 1024:
  (a) float route: per clip pcm.astype(float) / 32767 on the host, separate_channels, (stems * 32767) to int16 on the
      host in fp64 (the loop of examples/_common.py for --keep-channels on more than two channels);
  (b) separate_pcm16_channels_batch on all twelve clips in one call;
  (c) the same with wiener=2, wiener_radius=0;
  (d) the same with wiener=2, wiener_radius=2.
(a) and (b) are alternated, then (c) and (d), after one warm-up round; host wall clock around each route, ending in a
device synchronise, as audio-seconds per second (medians and ranges).  Beside them: the bytes each route moves over the
host link, computed from the shapes, and the kernel time per clip on the launching stream -- CUDA events around
separate_channels on planes already on the device for (a), the dcs_profile scopes of the batch's decode + separation and
encode for (b) to (d) -- so that it shows whether the link or the kernels bound each route.  It reads the card's name,
power limit and max SM clock in the same run, and exits without a GPU.

    python tools/time_pcm16_channels.py [--reps 3] [--out results.json]
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
from time_channels import SR, card, clip, synth_params  # noqa: E402

NCH, NCLIPS, NSRC = 6, 12, 4


def pinned(shape, dtype):
    return torch.empty(shape, dtype=dtype, pin_memory=True).numpy()


def make_clips(seed=2024):
    """NCLIPS int16 [L, 6] clips of 60..180 s in pinned memory"""
    rng = np.random.default_rng(seed)
    out = []
    for k, s in enumerate(rng.uniform(60.0, 180.0, NCLIPS)):
        a = clip(float(s), NCH, seed=seed + k)                             # float32 planes [6, L]
        p = pinned((a.shape[1], NCH), torch.int16)
        p[...] = np.round(a.T * 32767 * 0.8).astype(np.int16)
        out.append(p)
    return out


def route_a(sep, clips, outs):
    for pcm, o in zip(clips, outs):
        stems = sep.separate_channels(pcm.astype("float") / 32767)                        # [L, nsrc, C]
        o[...] = (stems.transpose(1, 0, 2).astype(np.float64) * 32767).astype("int16")


def wall(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def summary(v, audio_s):
    r = [audio_s / t for t in v]
    return {"audio_s_per_s_median": float(np.median(r)), "min": float(np.min(r)), "max": float(np.max(r)),
            "wall_s": [float(t) for t in v]}


def kernel_ms_a(sep, clips):
    """per clip: CUDA events around separate_channels on device-resident planes (its kernels only)"""
    ms = []
    for pcm in clips:
        x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")
        o = torch.empty((NSRC * NCH, x.shape[1]), dtype=torch.float32, device="cuda")
        sep.separate_channels(x, o)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sep.separate_channels(x, o)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        del x, o
    return ms


def kernel_ms_batch(sep, clips, outs, **kw):
    """per clip: the dcs_profile scopes of the batch (decode + separation, encode), on the launching stream"""
    sep.ctx.profile(True)
    sep.separate_pcm16_channels_batch(clips, outs=outs, **kw)
    torch.cuda.synchronize()
    rec = sep.ctx.profile_read()
    sep.ctx.profile(False)
    dec = [ms for n, ms in rec if n == "pcm16_decode_separate"]
    enc = [ms for n, ms in rec if n == "pcm16_encode"]
    assert len(dec) == len(enc) == len(clips), (len(dec), len(enc))
    return [d + e for d, e in zip(dec, enc)], enc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_pcm16_channels.py measures on the GPU and found none")
    res = {"card": card(), "reps": args.reps, "channels": NCH, "configs": []}
    print(json.dumps(res["card"]), flush=True)
    clips = make_clips()
    Ls = [c.shape[0] for c in clips]
    audio_s = sum(Ls) / SR
    res["clip_seconds"] = [L / SR for L in Ls]
    samples = sum(Ls)
    res["link_MB"] = {"a_h2d_fp32": samples * NCH * 4 / 1e6, "a_d2h_fp32": samples * NCH * NSRC * 4 / 1e6,
                      "b_h2d_int16": samples * NCH * 2 / 1e6, "b_d2h_int16": samples * NCH * NSRC * 2 / 1e6}
    print(json.dumps({"audio_s": audio_s, "link_MB": res["link_MB"]}), flush=True)
    outs_a = [pinned((NSRC, L, NCH), torch.int16) for L in Ls]
    outs_b = [pinned((NSRC, L, NCH), torch.int16) for L in Ls]
    for N in (2048, 1024):
        sep = Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25)
        routes = {"a_float_route": lambda: route_a(sep, clips, outs_a),
                  "b_pcm16_batch": lambda: sep.separate_pcm16_channels_batch(clips, outs=outs_b),
                  "c_pcm16_batch_wiener2": lambda: sep.separate_pcm16_channels_batch(clips, outs=outs_b, wiener=2),
                  "d_pcm16_batch_wiener2_radius2": lambda: sep.separate_pcm16_channels_batch(clips, outs=outs_b, wiener=2,
                                                                                            wiener_radius=2)}
        for f in routes.values():
            wall(f)
        t = {k: [] for k in routes}
        for group in (("a_float_route", "b_pcm16_batch"), ("c_pcm16_batch_wiener2", "d_pcm16_batch_wiener2_radius2")):
            for _ in range(args.reps):
                for k in group:
                    t[k].append(wall(routes[k]))
        cfg = {"N": N, "routes": {k: summary(v, audio_s) for k, v in t.items()}}
        # (a) against (b) on the same clips: the host encodes in fp64, the device in fp32
        route_a(sep, clips, outs_a)
        sep.separate_pcm16_channels_batch(clips, outs=outs_b)
        diff = [int(np.count_nonzero(a != b)) for a, b in zip(outs_a, outs_b)]
        maxd = max(int(np.abs(a.astype(np.int32) - b.astype(np.int32)).max()) for a, b in zip(outs_a, outs_b))
        cfg["a_vs_b"] = {"differing_values": sum(diff), "of": samples * NCH * NSRC, "max_abs_diff": maxd}
        ka = kernel_ms_a(sep, clips)
        kb, kb_enc = kernel_ms_batch(sep, clips, outs_b)
        kc, _ = kernel_ms_batch(sep, clips, outs_b, wiener=2)
        kd, _ = kernel_ms_batch(sep, clips, outs_b, wiener=2, wiener_radius=2)
        cfg["kernel_ms_per_clip"] = {"a": ka, "b": kb, "b_encode": kb_enc, "c": kc, "d": kd}
        cfg["kernel_s_total"] = {k: sum(v) / 1e3 for k, v in (("a", ka), ("b", kb), ("c", kc), ("d", kd))}
        cfg["workspace_MB"] = sep.ctx.workspace_bytes() / 1e6
        res["configs"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del sep
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
