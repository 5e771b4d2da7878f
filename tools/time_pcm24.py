"""Host-to-host throughput of packed 24-bit PCM (engine.PCM24) against int32 carrying the same 24-bit values
(development aid, not the bench).

  (1) the clip set of tools/time_channels_formats.py (twelve seeded 6-channel clips of 60 to 180 s, pinned in and out)
      at 44.1 and 48 kHz, N = 2048 and 1024: Separator.separate_channels_batch with PCM24 in and out against int32 in
      and out, alternated after one warm-up round; the bytes each moves over the host link, from the shapes, and its
      kernel time per dcs_profile scope;
  (2) 30 min of 6-channel audio at 48 kHz (tools/time_long_channels.py's recording as 24-bit values), N = 2048:
      separate_long_channels (120 s segments) in PCM24 against int32, without the filter and with K = 2, W = 2;
  (3) the fused decode and encode (dcs_channels_decode / _encode with the resampler) of PCM24 against int32 on the
      longest 48 kHz clip, CUDA events, alternated;
  (4) file to stems in host memory for one 6-channel 24-bit WAV of the longest 48 kHz clip: util.wav_samples (a memmap
      of the data chunk, pageable) + the PCM24 batch, against scipy.io.wavfile.read + the int32 batch; stems into pinned
      buffers.  The file is written to a temporary directory first, so both read it from the page cache.
Host wall clock around each route, ending in a device synchronise, as audio-seconds per second (medians and ranges of
--reps).  It reads the card's name, power limit and max SM clock in the same run, and exits without a GPU.

    python tools/time_pcm24.py [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import scipy.io.wavfile  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200 import _lib, util  # noqa: E402
from deepconvsep_b200.engine import PCM24, Separator  # noqa: E402
from time_channels import card, synth_params  # noqa: E402
from time_channels_formats import kernel_scopes, med, signals, summary, wall  # noqa: E402
from time_long_channels import recording  # noqa: E402

MODEL = 44100
NCH, NSRC = 6, 4
FMTS = {"i24": (PCM24, _lib.SAMPLE_I24), "i32": (np.dtype(np.int32), _lib.SAMPLE_I32)}


def pinned(shape, dtype):
    """pinned host array; PCM24 as pinned bytes viewed as V3"""
    dtype = np.dtype(dtype)
    p = torch.empty(int(np.prod(shape)) * dtype.itemsize, dtype=torch.uint8, pin_memory=True).numpy()
    return p.view(dtype).reshape(shape)


def as_fmt(v24, fmt):
    """24-bit values [L, C] (int32 or int64) -> pinned [L, C] of fmt"""
    p = pinned(v24.shape, FMTS[fmt][0])
    if fmt == "i32":
        p[...] = (v24 << 8).astype(np.int32)
    else:
        u = (v24 & 0xFFFFFF).astype(np.uint32)
        b = p.view(np.uint8).reshape(v24.shape + (3,))
        b[..., 0], b[..., 1], b[..., 2] = u & 0xFF, (u >> 8) & 0xFF, u >> 16
    return p


def alternate(routes, reps):
    for f, _ in routes.values():
        wall(f)
    t = {k: [] for k in routes}
    for _ in range(reps):
        for k, (f, _) in routes.items():
            t[k].append(wall(f))
    return {k: summary(v, routes[k][1]) for k, v in t.items()}


def kernels(sep, pcm, fmt_codes, rate, reps):
    """fused decode / encode per format on one clip, CUDA events, alternated"""
    lib, h = sep.lib, sep.ctx.handle
    to, back = sep.resampler(rate, MODEL), sep.resampler(MODEL, rate)
    L = pcm["i32"].shape[0]
    Lm = to.length(L)
    d_in = {f: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).ravel().copy()).cuda() for f, a in pcm.items()}
    planes = torch.empty((NCH + 1, Lm), dtype=torch.float32, device="cuda")
    stems = torch.randn((NSRC * NCH, Lm), dtype=torch.float32, device="cuda") * 0.1
    d_out = torch.empty(NSRC * NCH * L * 4, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    runs = {}
    for f, code in fmt_codes.items():
        runs["decode_" + f] = (lambda f=f, code=code: _lib.check(lib.dcs_channels_decode(
            h, to.handle, code, d_in[f].data_ptr(), L, NCH, planes.data_ptr(), Lm, None)))
        runs["encode_" + f] = (lambda code=code: _lib.check(lib.dcs_channels_encode(
            h, back.handle, code, stems.data_ptr(), Lm, NSRC, NCH, Lm, d_out.data_ptr(), L, NCH * L, None)))
    t = {k: [] for k in runs}
    for f in runs.values():
        f()
    for _ in range(max(reps, 5)):
        for k, f in runs.items():
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            t[k].append(e0.elapsed_time(e1))
    return {k: med(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_pcm24.py measures on the GPU and found none")
    res = {"card": card(), "reps": args.reps, "channels": NCH, "batch": [], "long": [], "kernels": None, "file": None}
    print(json.dumps(res["card"]), flush=True)
    seps = {N: Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25) for N in (2048, 1024)}
    codes = {f: c for f, (_, c) in FMTS.items()}
    for rate in (MODEL, 48000):
        v24 = [np.round(x * 2 ** 23).astype(np.int64) for x in signals(rate)]
        Ls = [v.shape[0] for v in v24]
        audio_s = sum(Ls) / rate
        clips = {f: [as_fmt(v, f) for v in v24] for f in FMTS}
        outs = {f: [pinned((NSRC, L, NCH), FMTS[f][0]) for L in Ls] for f in FMTS}
        for N, sep in seps.items():
            routes = {f: (lambda f=f: sep.separate_channels_batch(clips[f], outs=outs[f], sample_rate=rate), audio_s)
                      for f in FMTS}
            cfg = {"rate": rate, "N": N, "audio_s": audio_s, "routes": alternate(routes, args.reps)}
            for f in FMTS:
                b = FMTS[f][0].itemsize
                cfg["routes"][f]["link_MB"] = sum(Ls) * NCH * b * (1 + NSRC) / 1e6
                cfg["routes"][f]["kernel_ms_by_scope"] = kernel_scopes(sep, clips[f], outs[f], rate)
            same = all(np.array_equal(a.view(np.uint8).reshape(-1, 3), o.view(np.uint8).reshape(-1, 4)[:, 1:])
                       for a, o in zip(outs["i24"], outs["i32"]))
            cfg["i24_is_i32_top_bytes"] = bool(same)
            res["batch"].append(cfg)
            print(json.dumps(cfg), flush=True)
        if rate == 48000:
            k = int(np.argmax(Ls))
            res["kernels"] = {"L": Ls[k], "ms": kernels(seps[2048], {f: clips[f][k] for f in FMTS}, codes, rate, args.reps)}
            print(json.dumps(res["kernels"]), flush=True)
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "clip24.wav")
                util.write_wav(path, rate, clips["i24"][k])
                sep = seps[2048]
                o24, o32 = pinned((NSRC, Ls[k], NCH), PCM24), pinned((NSRC, Ls[k], NCH), np.int32)

                def packed():
                    r, x = util.wav_samples(path)
                    sep.separate_channels_batch([x], outs=[o24], sample_rate=r)

                def scipy_int32():
                    r, x = scipy.io.wavfile.read(path)
                    sep.separate_channels_batch([x], outs=[o32], sample_rate=r)
                routes = {"wav_samples_i24": (packed, Ls[k] / rate), "scipy_read_i32": (scipy_int32, Ls[k] / rate)}
                res["file"] = {"file_MB": os.path.getsize(path) / 1e6, "audio_s": Ls[k] / rate,
                               "routes": alternate(routes, args.reps)}
            print(json.dumps(res["file"]), flush=True)
        del clips, outs
    sep = seps[2048]
    base = recording(1800.0, 48000, NCH).astype(np.int32) << 8          # 24-bit values
    rec = {f: as_fmt(base, f) for f in FMTS}
    del base
    L = rec["i32"].shape[0]
    outs = {f: pinned((NSRC, L, NCH), FMTS[f][0]) for f in FMTS}
    for K, W in ((0, 0), (2, 2)):
        routes = {f: (lambda f=f: sep.separate_long_channels(rec[f], out=outs[f], wiener=K, wiener_radius=W,
                                                              sample_rate=48000), L / 48000) for f in FMTS}
        cfg = {"seconds": 1800, "rate": 48000, "N": 2048, "wiener": K, "radius": W, "routes": alternate(routes, args.reps)}
        for f in FMTS:
            cfg["routes"][f]["link_MB"] = L * NCH * FMTS[f][0].itemsize * (1 + NSRC) / 1e6
        cfg["workspace_MB"] = sep.ctx.workspace_bytes() / 1e6
        res["long"].append(cfg)
        print(json.dumps(cfg), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
