"""Device timing of the C-channel Wiener post-filter (Separator.separate_channels(wiener=K, wiener_radius=W)) against
the same call without the filter (development aid, not the bench).

One seeded 180 s clip at N = 2048 with the DSD100 network: C = 6 without the filter alternated with K = 1, 2, 3 at
radius 0 and 2; C = 8 at K = 2; C = 2 through the new entry alternated with keep-channels with the filter (the same
2 x 2 kernels, a sanity check).  >= 10 timed calls each with CUDA events (medians and ranges), the dcs_profile times
of the filter's stages (wiener_init: the masked spectra and the first sums; wiener_em: the EM passes) of one call of
each, the workspace each call leaves, and the HBM and FP64 bounds of one EM pass computed from the shapes.  It reads
the card's name, power limit and max SM clock in the same run.

    python tools/time_wiener_channels.py [--reps 10] [--out results.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepconvsep_b200.engine import Separator  # noqa: E402
from time_channels import card, clip, stages, synth_params, timed  # noqa: E402


def em_bounds(T, ldf, F, nx, nsrc=4, hbm_tbs=3.35, fp64_tflops=34.0):
    """the least time of one EM pass: HBM (read nx X planes, read and write nsrc * nx stem planes) and FP64 (the
    algebra per (t, f): C from the R_j, its L D L^H factor, two substitutions, y_j = v_j R_j z, the partial sums)"""
    gb = (nx + 2 * nsrc * nx) * T * ldf * 8 / 1e9
    flop = nsrc * nx * nx * 2 + 8 * nx ** 3 / 3 + 8 * nx * nx + nsrc * (8 * nx * nx + 4 * nx * nx) + nsrc * 4 * nx
    return {"em_pass_gbytes": gb, "em_pass_hbm_ms": gb / hbm_tbs, "em_flop_per_tf": flop,
            "em_pass_fp64_ms": flop * T * F / (fp64_tflops * 1e12) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_wiener_channels.py measures on the GPU and found none")
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "N": 2048}
    print(json.dumps(res["card"]), flush=True)
    dev = torch.device("cuda", 0)
    x8 = torch.tensor(clip(args.seconds, 8), device=dev)
    x6, x2 = x8[:6].contiguous(), x8[:2].contiguous()
    L = x8.shape[1]
    N = 2048
    params = synth_params(N // 2 + 1)

    def make():
        return Separator(params, frame_size=N, hop=512, window="hanning", overlap=25)
    plain, filt, keep = make(), make(), make()
    o24, o32, o8 = (torch.empty((n, L), dtype=torch.float32, device=dev) for n in (24, 32, 8))
    T, ldf, F = plain.stft.num_frames(L), plain.stft.ldf, plain.stft.F
    calls = {"C6_plain": (plain, lambda: plain.separate_channels(x6, o24))}
    for W in (0, 2):
        for K in (1, 2, 3):
            calls["C6_K%d_W%d" % (K, W)] = (filt, lambda K=K, W=W: filt.separate_channels(x6, o24, wiener=K, wiener_radius=W))
    calls["C8_K2_W0"] = (filt, lambda: filt.separate_channels(x8, o32, wiener=2))
    calls["C2_K2_W0"] = (filt, lambda: filt.separate_channels(x2, o8, wiener=2))
    calls["keep_K2_W0"] = (keep, lambda: keep.separate_keep_channels(x2, o8, wiener=2))
    ms = {}
    for group in (("C6_plain", "C6_K1_W0", "C6_K2_W0", "C6_K3_W0"), ("C6_plain", "C6_K1_W2", "C6_K2_W2", "C6_K3_W2"),
                  ("C8_K2_W0",), ("C2_K2_W0", "keep_K2_W0")):
        ms.update(timed({k: calls[k][1] for k in group}, args.reps))
    prof, ws = {}, {}
    for k, (s, f) in calls.items():
        prof[k] = stages(s, f)
        fresh = make()
        g = {"C6_plain": lambda: fresh.separate_channels(x6, o24), "C8_K2_W0": lambda: fresh.separate_channels(x8, o32, wiener=2),
             "C2_K2_W0": lambda: fresh.separate_channels(x2, o8, wiener=2),
             "keep_K2_W0": lambda: fresh.separate_keep_channels(x2, o8, wiener=2)}.get(k)
        if g is None:
            K, W = int(k[4]), int(k[7])
            g = lambda K=K, W=W: fresh.separate_channels(x6, o24, wiener=K, wiener_radius=W)   # noqa: E731
        g()
        torch.cuda.synchronize()
        ws[k] = fresh.ctx.workspace_bytes()
        del fresh
        torch.cuda.empty_cache()
    res["configs"] = [{"name": k, "ms": ms[k], "stages_ms": prof[k], "workspace_mb": ws[k] / 1e6} for k in calls]
    res["bounds"] = {"C6": em_bounds(T, ldf, F, 6), "C8": em_bounds(T, ldf, F, 8), "C2": em_bounds(T, ldf, F, 2)}
    for c in res["configs"]:
        st = c["stages_ms"]
        print("%-12s median %8.2f ms  [%7.2f, %7.2f]  wiener_init %6.2f  wiener_em %6.2f  workspace %7.0f MB"
              % (c["name"], c["ms"]["median"], c["ms"]["min"], c["ms"]["max"], st.get("wiener_init", 0.0),
                 st.get("wiener_em", 0.0), c["workspace_mb"]), flush=True)
    print(json.dumps(res["bounds"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
