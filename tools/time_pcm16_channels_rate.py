"""Host-to-host throughput of 48 kHz 6-channel int16 wavs (development aid, not the bench): the host route the scripts
take with --resample --keep-channels against the int16 multi-clip scheduler at the clips' rate
(Separator.separate_pcm16_channels_batch(sample_rate=48000)).

The clip set of tools/time_pcm16_channels.py at 48 kHz: twelve seeded 6-channel int16 clips of 60 to 180 s in pinned host
memory, stems into pinned int16 buffers, the DSD100-shaped synthetic params of tools/time_channels.py, N = 2048 and 1024:
  (a) host route: per clip pcm.astype(float) / 32767 on the host, separate_channels(sample_rate=48000), (stems * 32767)
      to int16 on the host in fp64 (examples/_common.py with --resample --keep-channels on more than two channels);
  (b) separate_pcm16_channels_batch(sample_rate=48000) on all twelve clips in one call;
  (c) the same with wiener=2.
(a), (b) and (c) are alternated after one warm-up round; host wall clock around each route, ending in a device
synchronise, as audio-seconds per second (medians and ranges of --reps).  Beside them: the bytes each route moves over
the host link, from the shapes, and per clip the kernel time of (b) and (c) split by the dcs_profile scopes into
resample-decode, separation and resample-encode.

Then the two fused kernels against Resampler.resample on the same planes (the decode's C int16 channels against C fp32
planes to 44.1 kHz, the encode's nsrc*C stem planes against the same planes back), CUDA events, alternated: each
kernel's bytes from the shapes and their fraction of the HBM floor at 3.35 TB/s.  It reads the card's name, power limit
and max SM clock in the same run, and exits without a GPU.

    python tools/time_pcm16_channels_rate.py [--reps 3] [--out results.json]
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

RATE, MODEL = 48000, 44100
NCH, NCLIPS, NSRC = 6, 12, 4
HBM = 3.35e12                               # H100 SXM data-sheet HBM3 bandwidth, bytes/s


def pinned(shape, dtype):
    return torch.empty(shape, dtype=dtype, pin_memory=True).numpy()


def make_clips(seed=2024):
    """NCLIPS int16 [L, 6] clips of 60..180 s at RATE in pinned memory (time_channels.clip's signal, taken as RATE)"""
    rng = np.random.default_rng(seed)
    out = []
    for k, s in enumerate(rng.uniform(60.0, 180.0, NCLIPS)):
        a = clip(float(s) * RATE / MODEL, NCH, seed=seed + k)               # float32 planes [6, s * RATE]
        p = pinned((a.shape[1], NCH), torch.int16)
        p[...] = np.round(a.T * 32767 * 0.8).astype(np.int16)
        out.append(p)
    return out


def route_a(sep, clips, outs):
    for pcm, o in zip(clips, outs):
        stems = sep.separate_channels(pcm.astype("float") / 32767, sample_rate=RATE)        # [L, nsrc, C]
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


def kernel_ms_batch(sep, clips, outs, **kw):
    """per clip: the batch's dcs_profile scopes, on the launching stream"""
    sep.ctx.profile(True)
    sep.separate_pcm16_channels_batch(clips, outs=outs, sample_rate=RATE, **kw)
    torch.cuda.synchronize()
    rec = sep.ctx.profile_read()
    sep.ctx.profile(False)
    split = {k: [ms for n, ms in rec if n == k] for k in ("resample_decode", "pcm16_separate", "resample_encode")}
    assert all(len(v) == len(clips) for v in split.values()), {k: len(v) for k, v in split.items()}
    return split


def med(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def kernels_vs_resample(sep, pcm, reps):
    """the fused kernels (profile scopes of a one-clip batch) against Resampler.resample on the same planes, alternated"""
    to, back = sep.resampler(RATE, MODEL), sep.resampler(MODEL, RATE)
    L = pcm.shape[0]
    Lm = to.length(L)
    x = torch.tensor(np.ascontiguousarray(pcm.T).astype(np.float32) / np.float32(32767), device="cuda")   # [C, L]
    y = torch.empty((NCH, Lm), dtype=torch.float32, device="cuda")
    s = torch.randn((NSRC * NCH, Lm), dtype=torch.float32, device="cuda") * 0.1
    z = torch.empty((NSRC * NCH, L), dtype=torch.float32, device="cuda")
    out = [pinned((NSRC, L, NCH), torch.int16)]
    t = {"decode_fused": [], "resample_in": [], "encode_fused": [], "resample_back": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def ev(f):
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    to.resample(x, out=y)
    back.resample(s, num_out=L, out=z)
    for _ in range(reps):
        k = kernel_ms_batch(sep, [pcm], out)
        t["decode_fused"].append(k["resample_decode"][0])
        t["encode_fused"].append(k["resample_encode"][0])
        t["resample_in"].append(ev(lambda: to.resample(x, out=y)))
        t["resample_back"].append(ev(lambda: back.resample(s, num_out=L, out=z)))
    nbytes = {"decode_fused": 2 * NCH * L + 4 * (NCH + 1) * Lm, "resample_in": 4 * NCH * L + 4 * NCH * Lm,
              "encode_fused": 4 * NSRC * NCH * Lm + 2 * NSRC * NCH * L, "resample_back": 4 * NSRC * NCH * (Lm + L)}
    res = {}
    for k, v in t.items():
        m = float(np.median(v))
        res[k] = {"ms": med(v), "bytes": nbytes[k], "hbm_floor_fraction": nbytes[k] / HBM / (m / 1e3)}
    # what the fusion removes against decode -> dcs_resample -> downmix and dcs_resample -> encode, from the shapes
    res["unfused_extra_bytes"] = 4 * NCH * L + 4 * NCH * L + 4 * NCH * Lm + 8 * NSRC * NCH * L
    res["clip_samples"] = L
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_pcm16_channels_rate.py measures on the GPU and found none")
    res = {"card": card(), "reps": args.reps, "rate": RATE, "channels": NCH, "configs": []}
    print(json.dumps(res["card"]), flush=True)
    clips = make_clips()
    Ls = [c.shape[0] for c in clips]
    samples = sum(Ls)
    audio_s = samples / RATE
    res["clip_seconds"] = [L / RATE for L in Ls]
    res["link_MB"] = {"a_h2d_fp32": samples * NCH * 4 / 1e6, "a_d2h_fp32": samples * NCH * NSRC * 4 / 1e6,
                      "b_h2d_int16": samples * NCH * 2 / 1e6, "b_d2h_int16": samples * NCH * NSRC * 2 / 1e6}
    print(json.dumps({"audio_s": audio_s, "link_MB": res["link_MB"]}), flush=True)
    outs_a = [pinned((NSRC, L, NCH), torch.int16) for L in Ls]
    outs_b = [pinned((NSRC, L, NCH), torch.int16) for L in Ls]
    for N in (2048, 1024):
        sep = Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25)
        routes = {"a_host_route": lambda: route_a(sep, clips, outs_a),
                  "b_pcm16_batch": lambda: sep.separate_pcm16_channels_batch(clips, outs=outs_b, sample_rate=RATE),
                  "c_pcm16_batch_wiener2": lambda: sep.separate_pcm16_channels_batch(clips, outs=outs_b, wiener=2,
                                                                                    sample_rate=RATE)}
        for f in routes.values():
            wall(f)
        t = {k: [] for k in routes}
        for _ in range(args.reps):
            for k in routes:
                t[k].append(wall(routes[k]))
        cfg = {"N": N, "routes": {k: summary(v, audio_s) for k, v in t.items()}}
        route_a(sep, clips, outs_a)
        sep.separate_pcm16_channels_batch(clips, outs=outs_b, sample_rate=RATE)
        diff = [int(np.count_nonzero(a != b)) for a, b in zip(outs_a, outs_b)]
        maxd = max(int(np.abs(a.astype(np.int32) - b.astype(np.int32)).max()) for a, b in zip(outs_a, outs_b))
        cfg["a_vs_b"] = {"differing_values": sum(diff), "of": samples * NCH * NSRC, "max_abs_diff": maxd}
        for name, kw in (("b", {}), ("c", {"wiener": 2})):
            split = kernel_ms_batch(sep, clips, outs_b, **kw)
            cfg["kernel_ms_per_clip_" + name] = split
            cfg["kernel_s_total_" + name] = {k: sum(v) / 1e3 for k, v in split.items()}
        if N == 2048:
            longest = clips[int(np.argmax(Ls))]
            cfg["fused_vs_resample"] = kernels_vs_resample(sep, longest, max(args.reps, 3))
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
