"""Host-to-host throughput of 6-channel clips in int16, int32 (24-bit values) and float32 (development aid, not the
bench): the multi-clip scheduler (Separator.separate_channels_batch) against the host route of the same format, and
int16 through the old and the new entry point.

The clip set of tools/time_pcm16_channels.py: twelve seeded 6-channel clips of 60 to 180 s in pinned host memory, at
44.1 and 48 kHz, as int16 (0.8 of full scale), int32 (the same signal as 24-bit values in the top bytes) and float32
(the same signal), stems into pinned buffers of the same format; the DSD100-shaped synthetic params of
tools/time_channels.py, N = 2048 and 1024.  For each (format, rate, N), alternated after one warm-up round:
  (a) host route: per clip the host decode of the format (astype(float) / iinfo.max for the integers, the samples
      themselves for float32), separate_channels(sample_rate=rate), the host encode in fp64 (truncated, saturated for
      int32, the stems themselves for float32) -- on the first clip only, to bound the time it takes;
  (b) separate_channels_batch on all twelve clips in one call;
  (o) int16 only: separate_pcm16_channels_batch on the same clips, the entry point before the formats existed.
Host wall clock around each route, ending in a device synchronise, as audio-seconds per second (medians and ranges of
--reps).  Beside them: the bytes (b) moves over the host link, from the shapes, and the kernel time of (b) per
dcs_profile scope.

Then, on the longest 48 kHz clip at N = 2048, the fused 4-byte kernels against the unfused chain on the same clip:
dcs_channels_decode with the resampler against the plain decode at 48 kHz + Resampler.resample of the C planes +
dcs_downmix_f32, and dcs_channels_encode with the resampler against Resampler.resample of the stem planes + the plain
encode, CUDA events, alternated.  It reads the card's name, power limit and max SM clock in the same run, and exits
without a GPU.

    python tools/time_channels_formats.py [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200 import _lib  # noqa: E402
from deepconvsep_b200.engine import Separator  # noqa: E402
from time_channels import card, clip, synth_params  # noqa: E402

MODEL = 44100
NCH, NCLIPS, NSRC, HOST_CLIPS = 6, 12, 4, 1
FORMATS = {"i16": (np.int16, _lib.SAMPLE_I16), "i32": (np.int32, _lib.SAMPLE_I32), "f32": (np.float32, _lib.SAMPLE_F32)}


def pinned(shape, dtype):
    return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True).numpy()


def signals(rate, seed=2024):
    """NCLIPS float64 [L, 6] signals of 60..180 s at `rate` at 0.8 of full scale (time_channels.clip's signal)"""
    rng = np.random.default_rng(seed)
    return [clip(float(s) * rate / MODEL, NCH, seed=seed + k).T.astype(np.float64) * 0.8
            for k, s in enumerate(rng.uniform(60.0, 180.0, NCLIPS))]


def as_format(x, fmt):
    dt = FORMATS[fmt][0]
    p = pinned(x.shape, dt)
    if fmt == "i16":
        p[...] = np.round(x * 32767).astype(np.int16)
    elif fmt == "i32":
        p[...] = (np.round(x * 2 ** 23).astype(np.int64) * 256).astype(np.int32)
    else:
        p[...] = x.astype(np.float32)
    return p


def host_route(sep, clips, outs, fmt, rate):
    """the scripts' host route for the format: host decode, separate_channels at the rate, host encode in fp64"""
    for pcm, o in zip(clips, outs):
        x = pcm.astype("float") / np.iinfo(pcm.dtype).max if fmt != "f32" else pcm
        stems = sep.separate_channels(x, sample_rate=rate).transpose(1, 0, 2).astype(np.float64)   # [nsrc, L, C]
        if fmt == "i16":
            o[...] = (stems * 32767).astype("int16")
        elif fmt == "i32":
            o[...] = np.clip(np.trunc(np.nan_to_num(stems * 2147483647.0)), -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int32)
        else:
            o[...] = stems.astype(np.float32)


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


def med(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def kernel_scopes(sep, clips, outs, rate):
    """kernel ms summed over the clips, per dcs_profile scope of one batch call"""
    sep.ctx.profile(True)
    sep.separate_channels_batch(clips, outs=outs, sample_rate=rate)
    torch.cuda.synchronize()
    rec = sep.ctx.profile_read()
    sep.ctx.profile(False)
    out = {}
    for n, ms in rec:
        out[n] = out.get(n, 0.0) + ms
    return out


def fused_vs_unfused(sep, pcm, fmt, rate, reps):
    """the fused 4-byte kernels against the unfused chain on one clip, CUDA events, alternated"""
    lib, h = sep.lib, sep.ctx.handle
    code = FORMATS[fmt][1]
    to, back = sep.resampler(rate, MODEL), sep.resampler(MODEL, rate)
    L = pcm.shape[0]
    Lm = to.length(L)
    d_in = torch.from_numpy(np.ascontiguousarray(pcm).view(np.uint8).ravel().copy()).cuda()
    fused_planes = torch.empty((NCH + 1, Lm), dtype=torch.float32, device="cuda")
    plain_planes = torch.empty((NCH + 1, L), dtype=torch.float32, device="cuda")
    res_planes = torch.empty((NCH + 1, Lm), dtype=torch.float32, device="cuda")
    stems = torch.randn((NSRC * NCH, Lm), dtype=torch.float32, device="cuda") * 0.1
    back_planes = torch.empty((NSRC * NCH, L), dtype=torch.float32, device="cuda")
    d_out = torch.empty(NSRC * NCH * L * 4, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def ev(f):
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def dec_fused():
        _lib.check(lib.dcs_channels_decode(h, to.handle, code, d_in.data_ptr(), L, NCH, fused_planes.data_ptr(), Lm, None))

    def dec_unfused():
        _lib.check(lib.dcs_channels_decode(h, None, code, d_in.data_ptr(), L, NCH, plain_planes.data_ptr(), L, None))
        to.resample(plain_planes[1:], out=res_planes[1:])
        _lib.check(lib.dcs_downmix_f32(h, res_planes[1:].data_ptr(), NCH, Lm, Lm, res_planes.data_ptr(), None))

    def enc_fused():
        _lib.check(lib.dcs_channels_encode(h, back.handle, code, stems.data_ptr(), Lm, NSRC, NCH, Lm, d_out.data_ptr(), L,
                                           NCH * L, None))

    def enc_unfused():
        back.resample(stems, num_out=L, out=back_planes)
        _lib.check(lib.dcs_channels_encode(h, None, code, back_planes.data_ptr(), L, NSRC, NCH, L, d_out.data_ptr(), L,
                                           NCH * L, None))
    runs = {"decode_fused": dec_fused, "decode_unfused": dec_unfused, "encode_fused": enc_fused,
            "encode_unfused": enc_unfused}
    for f in runs.values():
        f()
    assert torch.equal(fused_planes.view(torch.int32), res_planes.view(torch.int32))      # the same bits
    t = {k: [] for k in runs}
    for _ in range(reps):
        for k, f in runs.items():
            t[k].append(ev(f))
    b = FORMATS[fmt][0]().itemsize
    nbytes = {"decode_fused": b * NCH * L + 4 * (NCH + 1) * Lm,
              "decode_unfused": b * NCH * L + 4 * (NCH + 1) * L + 4 * NCH * (L + Lm) + 4 * (NCH + 1) * Lm,
              "encode_fused": 4 * NSRC * NCH * Lm + b * NSRC * NCH * L,
              "encode_unfused": 4 * NSRC * NCH * (Lm + L) + 4 * NSRC * NCH * L + b * NSRC * NCH * L}
    return {k: {"ms": med(v), "bytes": nbytes[k]} for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_channels_formats.py measures on the GPU and found none")
    res = {"card": card(), "reps": args.reps, "channels": NCH, "host_route_clips": HOST_CLIPS, "configs": []}
    print(json.dumps(res["card"]), flush=True)
    seps = {N: Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25) for N in (2048, 1024)}
    for rate in (MODEL, 48000):
        xs = signals(rate)
        Ls = [x.shape[0] for x in xs]
        audio_s = sum(Ls) / rate
        host_s = sum(Ls[:HOST_CLIPS]) / rate
        for fmt in FORMATS:
            dt = FORMATS[fmt][0]
            clips = [as_format(x, fmt) for x in xs]
            outs = [pinned((NSRC, L, NCH), dt) for L in Ls]
            outs_a = [pinned((NSRC, L, NCH), dt) for L in Ls[:HOST_CLIPS]]
            b = np.dtype(dt).itemsize
            link = {"h2d_MB": sum(Ls) * NCH * b / 1e6, "d2h_MB": sum(Ls) * NCH * NSRC * b / 1e6}
            for N, sep in seps.items():
                routes = {"a_host_route": (lambda: host_route(sep, clips[:HOST_CLIPS], outs_a, fmt, rate), host_s),
                          "b_batch": (lambda: sep.separate_channels_batch(clips, outs=outs, sample_rate=rate), audio_s)}
                if fmt == "i16":
                    routes["o_pcm16_batch"] = (lambda: sep.separate_pcm16_channels_batch(clips, outs=outs, sample_rate=rate),
                                               audio_s)
                for f, _ in routes.values():
                    wall(f)
                t = {k: [] for k in routes}
                for _ in range(args.reps):
                    for k, (f, _) in routes.items():
                        t[k].append(wall(f))
                cfg = {"format": fmt, "rate": rate, "N": N, "audio_s": audio_s, "link": link,
                       "routes": {k: summary(v, routes[k][1]) for k, v in t.items()}}
                sep.separate_channels_batch(clips, outs=outs, sample_rate=rate)
                diff = [int(np.count_nonzero(a != o[:, :, :])) for a, o in zip(outs_a, outs[:HOST_CLIPS])]
                cfg["a_vs_b_differing_values"] = {"n": sum(diff), "of": sum(Ls[:HOST_CLIPS]) * NCH * NSRC}
                cfg["kernel_ms_by_scope"] = kernel_scopes(sep, clips, outs, rate)
                med_b = cfg["routes"]["b_batch"]["audio_s_per_s_median"]
                cfg["b_link_GB_per_s"] = (link["h2d_MB"] + link["d2h_MB"]) / 1e3 / (audio_s / med_b)
                if N == 2048 and rate != MODEL and fmt != "i16":
                    cfg["fused_vs_unfused"] = fused_vs_unfused(sep, clips[int(np.argmax(Ls))], fmt, rate, max(args.reps, 5))
                res["configs"].append(cfg)
                print(json.dumps(cfg), flush=True)
            del clips, outs, outs_a
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
