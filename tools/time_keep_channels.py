"""Device timing of the keep-channels mode of the DSD100 network against the mono call (development aid, not the bench).

One seeded 180 s stereo clip at N = 2048 and N = 1024: warm-up, then mono (the downmix) and keep-channels separation
alternated, >= 10 timed calls each with CUDA events; the dcs_profile stage breakdown of one call of each; the int16
batch path (host wall clock, one clip per call); and the mask stage's bytes and FLOPs from the shapes.

    python tools/time_keep_channels.py [--reps 12] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def mask_stage_shapes(N, L, hop=512, tc=30, overlap=25, nx=1):
    """bytes the mask stage must move and the GEMM FLOPs it issues (3xTF32: three tf32 products per fp32 product)"""
    T = (L + hop - 1) // hop + 2
    F = N // 2 + 1
    P = (T - tc - 1) // (tc - overlap) + 1
    m_tiles = (F + 127) // 128
    groups = (T + 7) // 8
    x_bytes = nx * T * F * 8
    s_bytes = 4 * nx * T * F * 8
    g_bytes = P * 3 * tc * 52 * 4                  # decoder activations, read by every 128-bin tile (mostly from L2)
    w_bytes = 50 * F * 4
    flops = 2 * (m_tiles * 128) * (groups * 144) * 56 * 3
    return {"frames": T, "bins": F, "x_read_GB": x_bytes / 1e9, "s_write_GB": s_bytes / 1e9,
            "compulsory_GB": (x_bytes + s_bytes + g_bytes + w_bytes) / 1e9, "g_reads_per_tile_GB": g_bytes * m_tiles / 1e9,
            "gemm_GFLOP": flops / 1e9}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "seconds": args.seconds, "reps": args.reps, "configs": []}
    print(json.dumps(res["card"]), flush=True)
    audio = stereo_clip(args.seconds)
    L = audio.shape[0]
    dev = torch.device("cuda", 0)
    x2 = torch.tensor(np.ascontiguousarray(audio.T), device=dev)
    xm = ((x2[0] + x2[1]) * 0.5).contiguous()          # the downmix expression of the keep-channels path
    pcm = np.round(audio * 32767).astype(np.int16)
    for N in (2048, 1024):
        sep = Separator(synth_params(N // 2 + 1), frame_size=N, hop=512, window="hanning", overlap=25)
        om = torch.empty((4, L), dtype=torch.float32, device=dev)
        ok = torch.empty((8, L), dtype=torch.float32, device=dev)
        runs = {"mono": lambda: sep.separate_device(xm, om), "keep": lambda: sep.separate_keep_channels(x2, ok)}
        for _ in range(3):
            for f in runs.values():
                f()
        torch.cuda.synchronize()
        ms = {k: [] for k in runs}
        launches = {}
        for _ in range(args.reps):
            for k, f in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n0 = sep.ctx.launch_count()
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                launches[k] = sep.ctx.launch_count() - n0
                ms[k].append(e0.elapsed_time(e1))
        prof = {k: stages(sep, f) for k, f in runs.items()}
        # int16 path, host wall clock per one-clip call (H2D + kernels + D2H)
        wall = {"mono": [], "keep": []}
        for _ in range(3):
            sep.separate_pcm16(pcm)
            sep.separate_pcm16(pcm, keep_channels=True)
        for _ in range(max(3, args.reps // 2)):
            t0 = time.perf_counter()
            sep.separate_pcm16(pcm)
            wall["mono"].append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            sep.separate_pcm16(pcm, keep_channels=True)
            wall["keep"].append((time.perf_counter() - t0) * 1e3)
        cfg = {"N": N, "launches": launches,
               "ms": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in ms.items()},
               "stages_ms": prof,
               "pcm16_wall_ms": {k: {"median": float(np.median(v)), "min": float(np.min(v))} for k, v in wall.items()},
               "mask_stage": {"mono": mask_stage_shapes(N, L, nx=1), "keep": mask_stage_shapes(N, L, nx=2)}}
        m0 = prof["mono"].get("dec_convT1_mask_xfade", float("nan"))
        m1 = prof["keep"].get("dec_convT1_mask_xfade", float("nan"))
        cfg["mask_stage_ratio_keep_over_mono"] = m1 / m0
        res["configs"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del sep
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
