"""Dataset-level separation runner = the `if not skip_sep:` branch of the reference's trainers
(examples/dsd100/trainCNN.py:285-335, examples/ikala/trainCNN.py:246-285, same shape for Bach10 /
hiphopss): walk the dataset directory, separate every mixture with util's zero-padded patcher and
the analysis window the features were computed with, write the stems with the input's bit depth
(util.writeAudioScipy, util.py:56-58).  The reference does this one file at a time inside the
training process; here the model stays resident on the GPU and the songs are sharded over the
GPUs of a box (one process per GPU, `torchrun`), with no collective on the data path.

    python -m deepconvsep_b200.runner --family dsd --db <DSD100/Mixtures> --out <dir> --model model.pkl
    python -m deepconvsep_b200.runner --family bach10_score --db <Bach10> --out <dir> --model model.pkl
    torchrun --nproc-per-node 8 -m deepconvsep_b200.runner --family dsd --db ... --out ... --model ...
"""
import argparse
import os
import numpy as np

from . import util
from .engine import Separator, check_stereo_options
from .models import load_model, FAMILY_DEFAULTS
from .score import score_melody
from .sharding import shard_clips, reduce_stats

# trainer settings: (frameSize, hop, window, overlap) -- dsd100/trainCNN.py:431,399; ikala/trainCNN.py:382;
# bach10/trainCNNbach10.py uses 4096 / blackmanharris
TRAINER = {
    "dsd": dict(frameSize=1024, hopSize=512, window="blackmanharris", overlap=25),
    "ikala": dict(frameSize=1024, hopSize=512, window="blackmanharris", overlap=20),
    "bach10": dict(frameSize=4096, hopSize=512, window="blackmanharris", overlap=25),
    # stereo / ILD trainer: transformFFT(frameSize=1024, hopSize=512, window=hanning), overlap 25
    # (dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:487, 438-441)
    "dsd_ild": dict(frameSize=1024, hopSize=512, window="hanning", overlap=25),
    # score-informed Bach10: transformFFT(4096, 512, blackmanharris), overlap 25 (trainCNNrwc.py:585-587,653); the
    # network (build_ca, 17 or 11 arrays, or build_ca_1x1, 22 arrays) is inferred from the parameter list
    "bach10_score": dict(frameSize=4096, hopSize=512, window="blackmanharris", overlap=25),
}
# scale_factor_test of the score-informed trainer (trainCNNrwc.py:600-603,672); the other trainers separate with 0.3
DEFAULT_SCALE = {"bach10_score": 0.2}
# the score-informed trainer's sources (spelling of the reference) and their score files <instrument>_b.txt
# (trainCNNrwc.py:361-362)
SCORE_SOURCES = ["bassoon", "clarinet", "saxphone", "violin"]
SCORE_MIDI = ["bassoon_b", "clarinet_b", "saxophone_b", "violin_b"]


def list_jobs(family, testdir, outdir):
    """[(input wav, [output wavs])] in the reference's directory conventions."""
    jobs = []
    if family == "dsd_ild":
        # --db is the DSD100 root here: <db>/Mixtures/<sub>/<song>/mixture.wav -> <out>/Sources/<sub>/<song>/<source>.wav
        # (trainCNN_ILD_DSD100.py:296-300, 329-343)
        src = FAMILY_DEFAULTS["dsd_ild"]["sources"]
        for sub in ("Dev", "Test"):
            d = os.path.join(testdir, "Mixtures", sub)
            if not os.path.isdir(d):
                continue
            for f in sorted(os.listdir(d)):
                if f.startswith('.'):
                    continue
                jobs.append((os.path.join(d, f, "mixture.wav"),
                             [os.path.join(outdir, "Sources", sub, f, s + ".wav") for s in src]))
    elif family == "dsd":
        src = FAMILY_DEFAULTS["dsd"]["sources"]
        for sub in ("Dev", "Test"):
            d = os.path.join(testdir, sub)
            if not os.path.isdir(d):
                continue
            for f in sorted(os.listdir(d)):
                if f.startswith('.'):
                    continue
                jobs.append((os.path.join(d, f, "mixture.wav"), [os.path.join(outdir, sub, f, s + ".wav") for s in src]))
    elif family == "bach10_score":
        # piece directories whose name starts with a digit, the four source wavs inside, stems <out>/<piece>-<source>.wav
        # (trainCNNrwc.py:357-416,646-647); the job's input is the piece directory
        for f in sorted(os.listdir(testdir)):
            d = os.path.join(testdir, f)
            if os.path.isdir(d) and f[0].isdigit():
                jobs.append((d, [os.path.join(outdir, f + "-" + s + ".wav") for s in SCORE_SOURCES]))
    elif family == "ikala":
        for f in sorted(os.listdir(testdir)):
            if f.endswith(".wav"):
                jobs.append((os.path.join(testdir, f), [os.path.join(outdir, f.replace(".wav", "-voice.wav")),
                                                        os.path.join(outdir, f.replace(".wav", "-music.wav"))]))
    else:
        src = FAMILY_DEFAULTS[family]["sources"]
        for f in sorted(os.listdir(testdir)):
            if f.endswith(".wav"):
                jobs.append((os.path.join(testdir, f), [os.path.join(outdir, f.replace(".wav", "_" + s + ".wav")) for s in src]))
    return jobs


def _num_samples(path):
    """Samples per channel from the wav header (memory-mapped, nothing is read); the shard balance and the
    longest-first order go by duration, not by bytes (a 24/32-bit song is not longer than a 16-bit one)."""
    import scipy.io.wavfile
    try:
        _, a = scipy.io.wavfile.read(path, mmap=True)
        return int(a.shape[0])
    except Exception:  # noqa: BLE001  (unreadable header: fall back to the byte count, the read itself will report)
        return int(os.path.getsize(path))


def _piece_sources(piece):
    name = os.path.basename(os.path.normpath(piece))
    return [os.path.join(piece, name + "-" + s + ".wav") for s in SCORE_SOURCES]


def read_piece(piece):
    """A Bach10 piece directory -> (mixture float64 [L] = the float sum of its four source wavs, sampleRate, bit depth)
    (trainCNNrwc.py:367-378)."""
    audio = None
    for path in _piece_sources(piece):
        audioObj, sampleRate, bitrate = util.readAudioScipy(path)
        assert sampleRate == 44100, "Sample rate needs to be 44100"
        audio = audioObj if audio is None else audio + audioObj
    return audio, sampleRate, bitrate


def _write_stems(paths, stems, sampleRate, bitrate):
    """stems[i] (float [nsamples] or [nsamples, 2]) -> the wav paths[i] at the input's bit depth."""
    for path, stem in zip(paths, stems):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        util.writeAudioScipy(path, stem.astype(np.float64), sampleRate, bitrate)


def _first_channels(jobs):
    """Channel count of the first mixture from its wav header; None where there is none to read."""
    try:
        import scipy.io.wavfile
        a = scipy.io.wavfile.read(jobs[0][0], mmap=True)[1]
        return 1 if a.ndim == 1 else int(a.shape[1])
    except Exception:  # noqa: BLE001
        return None


def separate_dataset(family, testdir, outdir, model, scale_factor=None, time_context=30, rank=0, world_size=1, device=0,
                     keep_channels=False, wiener=0, wiener_radius=0, **overrides):
    """scale_factor: None = the family's trainer value (0.2 for bach10_score, else 0.3).
    bach10_score: every piece directory of `testdir` (name starting with a digit): the mixture is the sum of its four
    source wavs, the note table comes from its <instrument>_b.txt scores (40 s window, 20 harmonics, +-50 cents,
    440 Hz) and the filters are rasterised from it on the GPU (Separator.separate_notes).
    keep_channels (family dsd): 2-channel stems in the same layout -- the soft masks of the downmix applied to each
    channel of the mixture (Separator.separate_keep_channels), so that a multichannel evaluation scores real stereo
    images.  wiener (family dsd with keep_channels, or dsd_ild): that many EM iterations of the multichannel Wiener
    post-filter on the stereo stems; wiener_radius: its covariance window in chunks of 128 frames to either side
    (0 = the whole song).  keep_channels on mixtures of C > 2 channels (any single-channel family; the first mixture
    decides): C-channel stems, the masks of the mean of the channels applied to each (Separator.separate_channels)."""
    nch = _first_channels(list_jobs(family, testdir, outdir)) if keep_channels and family != "bach10_score" else None
    check_stereo_options(family, keep_channels, wiener, wiener_radius, channels=nch if nch and nch > 2 else None)
    wkw = {"wiener": wiener} if wiener else {}
    if wiener_radius:
        wkw["wiener_radius"] = wiener_radius
    cfg = dict(TRAINER[family], **overrides)
    if scale_factor is None:
        scale_factor = DEFAULT_SCALE.get(family, 0.3)
    params = load_model(model) if isinstance(model, str) else model
    sep = Separator(params, arch=None if family in ("ikala", "bach10_score") else family, frame_size=cfg["frameSize"],
                    hop=cfg["hopSize"], window=cfg["window"], scale_factor=scale_factor, time_context=time_context,
                    overlap=cfg["overlap"], patcher="util", device=device, feat_size=cfg["frameSize"] // 2 + 1)
    if family == "bach10_score" and sep.model.arch not in ("bach10_score", "bach10_score_1x1"):
        raise ValueError("--family bach10_score needs a score-informed network, %s holds a %r network" % (
            model if isinstance(model, str) else "the parameter list", sep.model.arch))
    jobs = list_jobs(family, testdir, outdir)
    sizes = [_num_samples(_piece_sources(j[0])[0] if family == "bach10_score" else j[0]) for j in jobs]
    seconds = 0.0
    # longest first: the workspace buffers only grow, so the first song sizes them once for the whole shard
    for idx in sorted(shard_clips(sizes, world_size, rank), key=lambda i: (-sizes[i], i)):
        wav, outs = jobs[idx]
        if family == "bach10_score":
            audio, sampleRate, bitrate = read_piece(wav)
            nframes = int(np.ceil(len(audio) / np.double(cfg["hopSize"]))) + 2
            melody = score_melody(wav, SCORE_MIDI, nframes, frameSize=cfg["frameSize"], hopSize=cfg["hopSize"],
                                  sampleRate=sampleRate)
            stems = sep.separate_notes(audio, melody)
        else:
            audio, sampleRate, bitrate = util.readAudioScipy(wav)
            assert sampleRate == 44100, "Sample rate needs to be 44100"
            if keep_channels and audio.ndim == 2 and audio.shape[1] > 2:     # C channels in, C-channel stems out
                check_stereo_options(family, True, wiener, wiener_radius, channels=audio.shape[1])
                stems = sep.separate_channels(audio).transpose(1, 0, 2)
            elif family == "dsd_ild" or keep_channels:             # both channels in, stereo stems out
                assert audio.ndim == 2 and audio.shape[1] == 2, "%s needs 2-channel mixtures" % (
                    "--keep-channels" if keep_channels else "the stereo / ILD network")
                stereo = sep.separate_keep_channels(audio, **wkw) if keep_channels else sep.separate_stereo(audio, **wkw)
                stems = stereo.transpose(1, 0, 2)                  # [nsamples, nsrc, 2] -> [nsrc, nsamples, 2]
            else:
                if audio.ndim > 1:                                  # ikala/trainCNN.py:255, dsd100/trainCNN.py:304
                    audio = audio[:, 0] + audio[:, 1] if family == "ikala" else (audio[:, 0] + audio[:, 1]) / 2
                stems = sep.separate(audio)
        _write_stems(outs, stems, sampleRate, bitrate)
        seconds += len(audio) / float(sampleRate)
    return seconds, len(jobs)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--family", required=True, choices=sorted(TRAINER))
    ap.add_argument("--db", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--model", required=True)
    ap.add_argument("--scale-factor", type=float, default=None,
                    help="magnitude scale of the network input (default: 0.2 for --family bach10_score, else 0.3)")
    ap.add_argument("--keep-channels", action="store_true",
                    help="--family dsd: 2-channel stems, the soft masks of the downmix applied to each channel; mixtures of "
                         "more than 2 channels, any single-channel family: stems of as many channels")
    ap.add_argument("--wiener", type=int, default=0, metavar="K",
                    help="K EM iterations of the multichannel Wiener post-filter on the stereo stems "
                         "(--family dsd --keep-channels, or --family dsd_ild)")
    ap.add_argument("--wiener-radius", type=int, default=0, metavar="R",
                    help="with --wiener: spatial covariances over a sliding window of R chunks of 128 frames to either "
                         "side (default 0: one per song)")
    args = ap.parse_args(argv)
    nch = None
    if args.keep_channels and args.family != "bach10_score" and os.path.isdir(args.db):
        nch = _first_channels(list_jobs(args.family, args.db, args.out))
    try:
        check_stereo_options(args.family, args.keep_channels, args.wiener, args.wiener_radius,
                             channels=nch if nch and nch > 2 else None)
    except ValueError as e:
        ap.error(str(e))
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (("WORLD_SIZE", "1"), ("RANK", "0"), ("LOCAL_RANK", "0")))
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import time
    t0 = time.time()
    secs, njobs = separate_dataset(args.family, args.db, args.out, args.model, args.scale_factor, rank=rank,
                                   world_size=world, device=local, keep_channels=args.keep_channels,
                                   wiener=args.wiener, wiener_radius=args.wiener_radius)
    tot, ms, _ = reduce_stats(secs, (time.time() - t0) * 1e3)
    if rank == 0:
        print("separated %d files, %.1f audio-s in %.2f s (%.0f x real time) on %d GPU(s)" % (njobs, tot, ms / 1e3,
                                                                                          tot / (ms / 1e3), world))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
