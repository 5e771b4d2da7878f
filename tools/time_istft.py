"""Device timing of the inverse STFT + overlap-add (K4) on its own (development aid, not the bench).

For a 180 s clip, hop 512, at N = 2048 and N = 1024: the plain K4 on four spectra planes (dcs_istft) and the masked
K4 on one mixture STFT and four float masks (dcs_istft_masked, nx = 1), alternated, each timed with CUDA events;
medians over --reps launches, the algorithmic bytes and GB/s, and the card's name, power limit and maximum SM clock read
in the same run.  The masked result is also compared with the plain K4 on the same M * X (bit for bit).

    python tools/time_istft.py [--reps 21] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Context, Stft  # noqa: E402

SR = 44100


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, sm_max = [v.strip() for v in q.split(",")]
    except Exception:  # noqa: BLE001
        power, sm_max = None, None
    return {"gpu": name, "power_limit_w": power, "sm_max_mhz": sm_max}


def time_call(f, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def one_size(ctx, N, hop, seconds, reps, nsrc=4):
    dev = torch.device("cuda", 0)
    stft = Stft(ctx, N, hop)
    L = int(round(seconds * SR))
    T, ldf, F = stft.num_frames(L), stft.ldf, N // 2 + 1
    g = torch.Generator(device=dev).manual_seed(N + hop)
    X = torch.complex(torch.randn((1, T, ldf), device=dev, generator=g), torch.randn((1, T, ldf), device=dev, generator=g))
    M = torch.rand((nsrc, T, ldf), device=dev, generator=g)
    S = (M * X).contiguous()       # complex64 * float32: the same lone rounded products the masked kernel forms
    out_p = torch.empty((nsrc, L), dtype=torch.float32, device=dev)
    out_m = torch.empty((nsrc, L), dtype=torch.float32, device=dev)
    lib = ctx.lib
    from deepconvsep_b200 import _lib
    from deepconvsep_b200.engine import _ptr

    def plain():
        _lib.check(lib.dcs_istft(stft.handle, _ptr(S), nsrc, T, ldf, T * ldf, _ptr(out_p), L, L, None))

    def masked():
        _lib.check(lib.dcs_istft_masked(stft.handle, _ptr(X), 1, X.stride(0), _ptr(M), nsrc, M.stride(0), T, ldf,
                                        _ptr(out_m), L, L, None))
    for _ in range(3):
        plain()
        masked()
    torch.cuda.synchronize()
    tp, tm = [], []
    for _ in range(reps):          # alternated: both see the same state of the shared machine
        tp += time_call(plain, 1)
        tm += time_call(masked, 1)
    bytes_p = nsrc * T * F * 8 + nsrc * L * 4
    bytes_m = T * F * 8 + nsrc * T * F * 4 + nsrc * L * 4
    mp, mm = float(np.median(tp)), float(np.median(tm))
    res = {"N": N, "hop": hop, "frames": T, "samples": L, "nsrc": nsrc,
           "plain": {"ms_median": mp, "ms_min": float(np.min(tp)), "bytes": bytes_p, "gbps": bytes_p / (mp * 1e-3) / 1e9},
           "masked": {"ms_median": mm, "ms_min": float(np.min(tm)), "bytes": bytes_m, "gbps": bytes_m / (mm * 1e-3) / 1e9},
           "masked_equals_plain": bool(torch.equal(out_p, out_m))}
    stft.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--hop", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "sizes": []}
    print(json.dumps(res["card"]), flush=True)
    ctx = Context(0)
    for N in (2048, 1024):
        r = one_size(ctx, N, args.hop, args.seconds, args.reps)
        res["sizes"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
