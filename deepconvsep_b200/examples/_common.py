"""Shared driver of the stand-alone separation scripts: `train_auto` of
examples/dsd100/separate_dsd.py:239-313 (and its iKala / Bach10 siblings) on the CUDA pipeline."""
import os
import threading
import numpy as np
import scipy.io.wavfile

from ..engine import MODEL_RATE, Separator, check_resample_rates, check_stereo_options
from ..models import load_model, FAMILY_DEFAULTS

_cache = {}
_cache_lock = threading.Lock()       # run_many's worker threads share the cache


def get_separator(model, arch, frame_size, hop, window, scale_factor, time_context, overlap, feat_size, device=0, slot=0):
    key = (os.path.abspath(model), os.path.getmtime(model), arch, frame_size, hop, str(window), scale_factor,
           time_context, overlap)
    with _cache_lock:
        if _cache.get("key") != key:
            _cache.clear()   # one resident model at a time (Bach10 weights are 856 MB), per (device, slot)
            _cache["key"] = key
        if (device, slot) not in _cache:
            _cache[(device, slot)] = Separator(load_model(model), arch=arch, frame_size=frame_size, hop=hop, window=window,
                                               scale_factor=scale_factor, time_context=time_context, overlap=overlap,
                                               patcher="standalone", feat_size=feat_size, device=device)
        return _cache[(device, slot)]


def decode(audioObj, family):
    """scipy.io.wavfile array -> mono float in the reference's (quirky) normalisation:
    divide by iinfo.max -- or by finfo.max for float wavs, which makes those silent
    (separate_dsd.py:277-287; SURVEY.md 0.9) -- then (L+R)/2, or L+R for iKala."""
    if np.issubdtype(audioObj.dtype, np.floating):
        maxv = np.finfo(audioObj.dtype).max
    else:
        maxv = np.iinfo(audioObj.dtype).max
    a = audioObj.astype('float') / maxv
    if family == "ikala":
        return a[:, 0] + a[:, 1]                 # separate_ikala.py:229 (needs a stereo file)
    if a.ndim > 1 and a.shape[1] > 1:
        return (a[:, 0] + a[:, 1]) / 2
    return a if a.ndim == 1 else a[:, 0]


def wav_channels(path):
    """Channel count of a wav, or of the first wav of a directory, from the header (memory-mapped: nothing is read);
    None where there is none to read."""
    try:
        if os.path.isdir(path):
            path = sorted(os.path.join(path, f) for f in os.listdir(path) if f.lower().endswith(".wav"))[0]
        a = scipy.io.wavfile.read(path, mmap=True)[1]
        return 1 if a.ndim == 1 else int(a.shape[1])
    except Exception:  # noqa: BLE001  (unreadable: the read in run() reports it)
        return None


def wav_rate(path):
    """Sample rate of a wav from its header (memory-mapped: nothing else is read); None where there is none to read."""
    try:
        return int(scipy.io.wavfile.read(path, mmap=True)[0])
    except Exception:  # noqa: BLE001  (unreadable: the read in run() reports it)
        return None


def _one_over_devices_at_rate(filein, rate):
    return ("--resample: %s is at %d Hz, and one recording at a rate other than 44100 Hz runs on one device; cutting it "
            "over several is not implemented (a directory of wavs goes over the devices file by file)" % (filein, rate))


def run(family, filein, outdir, model, scale_factor, time_context, overlap, batch_size, input_size, frame_size, hop,
        out_name, window=None, device=0, slot=0, keep_channels=False, wiener=0, wiener_radius=0, resample=False):
    """wav in -> one int16 wav per source in `outdir`.  `batch_size` is accepted for signature
    compatibility; the CUDA path has no patch batches.  keep_channels (DSD100 / hiphopss, 2-channel wav): one
    2-channel wav per source -- the soft masks of the downmix applied to each channel; wiener: that many EM iterations
    of the multichannel Wiener post-filter on them (keep_channels only), wiener_radius: its covariance window in chunks
    to either side (0 = the whole clip).  keep_channels on a wav of C > 2 channels (5.1, arrays; every single-channel
    family): one C-channel wav per source, the masks of the mean of the channels applied to each
    (Separator.separate_channels; no Wiener filter, one device).  A device list cuts the recording into segments over the devices; with
    keep_channels and wiener that needs wiener_radius >= 1.  resample: a wav at another rate than 44100 Hz is separated
    through the float Separator calls with sample_rate= (resampled to 44.1 kHz and back on the device, one device) and its
    stems are written at the wav's rate and length; without it such a wav is reported and skipped, as by the reference."""
    nch = wav_channels(filein) if keep_channels else None
    if nch == 1:
        raise ValueError("--keep-channels needs at least a 2-channel recording; %s has 1 channel" % (filein,))
    check_stereo_options(family, keep_channels, wiener, wiener_radius, channels=nch)
    wkw = {"wiener": wiener} if wiener else {}
    if wiener_radius:
        wkw["wiener_radius"] = wiener_radius
    d = dict(FAMILY_DEFAULTS[family])
    if window is not None:
        d["window"] = window
    sampleRate, audioObj = scipy.io.wavfile.read(filein)
    if sampleRate != 44100 and not resample:
        print("Sample rate is not 44100")        # separate_dsd.py:313
        return None
    arch = None if family in ("ikala",) else family
    if sampleRate != 44100:
        if isinstance(device, (list, tuple)):
            if len(device) > 1:
                raise ValueError(_one_over_devices_at_rate(filein, sampleRate))
            device = device[0]
        check_resample_rates(sampleRate, MODEL_RATE)        # a rate it cannot take is refused before the model loads
        sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                            device=device, slot=slot)
        if keep_channels:
            maxv = np.finfo(audioObj.dtype).max if np.issubdtype(audioObj.dtype, np.floating) else np.iinfo(audioObj.dtype).max
            audio = audioObj.astype('float') / maxv
            if audioObj.shape[1] > 2:
                stems = sep.separate_channels(audio, sample_rate=sampleRate)                # [L, nsrc, C]
            else:
                stems = sep.separate_keep_channels(audio, sample_rate=sampleRate, **wkw)    # [L, nsrc, 2]
            stems16 = (stems.transpose(1, 0, 2).astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
        else:
            stems = sep.separate(decode(audioObj, family), sample_rate=sampleRate)
            stems16 = (stems.astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
    elif keep_channels:
        maxv = np.finfo(audioObj.dtype).max if np.issubdtype(audioObj.dtype, np.floating) else np.iinfo(audioObj.dtype).max
        if audioObj.shape[1] > 2:
            if isinstance(device, (list, tuple)):
                if len(device) > 1:
                    raise ValueError("--keep-channels on %d channels runs on one device; cutting such a recording over "
                                     "several is not implemented" % audioObj.shape[1])
                device = device[0]
            sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                                device=device, slot=slot)
            stems = sep.separate_channels(audioObj.astype('float') / maxv)              # [L, nsrc, C]
            stems16 = (stems.transpose(1, 0, 2).astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
        elif isinstance(device, (list, tuple)):
            # one stereo recording over several GPUs: segments on the chunk grid of the Wiener filter's windows
            from .. import longclip
            seps = [get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                                  device=dev, slot=slot) for dev in device]
            sep = seps[0]
            stems = longclip.separate_long(seps, audioObj.astype('float') / maxv, keep_channels=True, **wkw)
            stems16 = (stems.transpose(1, 0, 2).astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
        elif audioObj.dtype == np.int16:
            sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                                device=device, slot=slot)
            stems16 = sep.separate_pcm16(audioObj, keep_channels=True, **wkw)      # [nsrc, L, 2], int16 path on the GPU
        else:
            sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                                device=device, slot=slot)
            stems = sep.separate_keep_channels(audioObj.astype('float') / maxv, **wkw)    # [L, nsrc, 2]
            stems16 = (stems.transpose(1, 0, 2).astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
    elif isinstance(device, (list, tuple)):
        # one recording over several GPUs: hop- and patch-aligned segments with margins, one host thread per device,
        # the stitched stems are those of the whole-clip call (deepconvsep_b200.longclip)
        from .. import longclip
        seps = [get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                              device=dev, slot=slot) for dev in device]
        sep = seps[0]
        stems = longclip.separate_long(seps, decode(audioObj, family))
        stems16 = (stems.astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
    elif audioObj.dtype == np.int16 and family != "ikala":
        sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                            device=device, slot=slot)
        stems16 = sep.separate_pcm16(audioObj, downmix=1)          # decode/downmix/encode on the GPU
    else:
        sep = get_separator(model, arch, frame_size, hop, d["window"], scale_factor, time_context, overlap, input_size,
                            device=device, slot=slot)
        audio = decode(audioObj, family)
        stems = sep.separate(audio)
        stems16 = (stems.astype(np.float64) * np.iinfo(np.int16).max).astype('int16')
    _, filename = os.path.split(filein)
    paths = []
    for i, name in enumerate(sep.sources):
        path = os.path.join(outdir, out_name(filename, name))
        scipy.io.wavfile.write(filename=path, rate=sampleRate, data=stems16[i])
        paths.append(path)
    return paths


# ---- command line shared by the separate_*.py scripts ------------------------------------------------------
LONG_OPTS = ["ifile=", "odir=", "mfile=", "frame-size=", "window=", "devices=", "batch-clips=", "keep-channels", "wiener=",
             "wiener-radius=", "resample"]
EXTRA_USAGE = ("  optional: --frame-size N (STFT frame, feat_size = N/2+1)  --window hanning|blackmanharris|sinebell\n"
               "            --devices 0,1,...  --batch-clips K (clips in flight per device); with these, -i may be a directory of wavs\n"
               "            (one wav and several devices: the recording itself is cut into segments over the devices)\n"
               "            --keep-channels (DSD100 / hiphopss, 2-channel wavs): 2-channel stems, the downmix's masks on each channel;\n"
               "            on wavs of more than 2 channels (5.1, arrays), for every script: stems of as many channels\n"
               "            --wiener K (with --keep-channels): K EM iterations of the multichannel Wiener post-filter on them\n"
               "            --wiener-radius R (with --wiener): covariances over a window of R chunks of 128 frames to either\n"
               "            side instead of the whole clip; needed to cut one recording over several devices with --wiener\n"
               "            --resample: wavs at other rates (8 to 192 kHz, e.g. 48000, 96000) are resampled to 44.1 kHz and\n"
               "            back on the GPU and their stems written at their own rate and length (one wav: one device)")


def parse_cli(argv, usage):
    """getopt like the reference scripts (`-i -o -m`, separate_dsd.py:316-332) plus the long options SURVEY.md 5 asks for."""
    import getopt
    import sys
    try:
        opts, _ = getopt.getopt(argv, "hi:o:m:", LONG_OPTS)
    except getopt.GetoptError:
        print(usage)
        print(EXTRA_USAGE)
        sys.exit(2)
    o = {"inputfile": None, "outdir": None, "model": None, "frame_size": None, "window": None, "devices": None, "batch_clips": 1,
         "keep_channels": False, "wiener": 0, "wiener_radius": 0, "resample": False}
    for opt, arg in opts:
        if opt == "-h":
            print(usage)
            print(EXTRA_USAGE)
            sys.exit()
        elif opt in ("-i", "--ifile"):
            o["inputfile"] = arg
        elif opt in ("-o", "--odir"):
            o["outdir"] = arg
        elif opt in ("-m", "--mfile"):
            o["model"] = arg
        elif opt == "--frame-size":
            o["frame_size"] = int(arg)
        elif opt == "--window":
            o["window"] = arg
        elif opt == "--devices":
            o["devices"] = [int(x) for x in arg.split(",") if x != ""]
        elif opt == "--batch-clips":
            o["batch_clips"] = max(1, int(arg))
        elif opt == "--keep-channels":
            o["keep_channels"] = True
        elif opt == "--wiener":
            o["wiener"] = int(arg)
        elif opt == "--wiener-radius":
            o["wiener_radius"] = int(arg)
        elif opt == "--resample":
            o["resample"] = True
    if o["inputfile"] is None or o["outdir"] is None or o["model"] is None:
        print(usage)
        sys.exit(2)
    return o


def cli_main(argv, usage, train_auto_default, run_one, family=None):
    """`train_auto_default(inputfile, outdir, model)` = the script's literal reference call (no extra flag given);
    `run_one(filein, outdir, model, frame_size, window, device, slot, several_clips)` = the same with the overrides
    (with --keep-channels also keep_channels=True, wiener=K with --wiener K and wiener_radius=R with --wiener-radius R;
    only the DSD100 / hiphopss script, family "dsd", takes them; with --resample also resample=True)."""
    import sys
    o = parse_cli(argv, usage)
    # more than 2 channels (of the wav, or of the first wav of a directory) widens --keep-channels to every
    # single-channel family; a 1-channel file is reported by run(), with its name
    nch = wav_channels(o["inputfile"]) if o["keep_channels"] else None
    try:
        check_stereo_options(family, o["keep_channels"], o["wiener"], o["wiener_radius"], channels=nch if nch and nch > 2 else None)
    except ValueError as e:
        sys.exit(str(e))
    one_over_devices = not os.path.isdir(o["inputfile"]) and len(o["devices"] or []) > 1
    if o["wiener"] and not o["wiener_radius"] and one_over_devices:
        sys.exit("--wiener %d over several devices needs --wiener-radius R >= 1: the recording is cut into segments, and "
                 "whole-clip covariances (wiener_radius 0) need the whole recording in one" % o["wiener"])
    if o["resample"] and one_over_devices and wav_rate(o["inputfile"]) not in (None, 44100):
        sys.exit(_one_over_devices_at_rate(o["inputfile"], wav_rate(o["inputfile"])))
    kw = {"resample": True} if o["resample"] else {}
    if o["keep_channels"]:
        kw["keep_channels"] = True
        if o["wiener"]:
            kw["wiener"] = o["wiener"]
        if o["wiener_radius"]:
            kw["wiener_radius"] = o["wiener_radius"]
    if kw:
        base = run_one

        def run_one(*args):
            return base(*args, **kw)
    plain = o["frame_size"] is None and o["window"] is None and o["devices"] is None and o["batch_clips"] == 1 \
        and not os.path.isdir(o["inputfile"])
    if plain and kw:
        return run_one(o["inputfile"], o["outdir"], o["model"], None, None, 0, 0, False)
    if plain:
        return train_auto_default(o["inputfile"], o["outdir"], o["model"])
    if os.path.isdir(o["inputfile"]):
        files = sorted(os.path.join(o["inputfile"], f) for f in os.listdir(o["inputfile"]) if f.lower().endswith(".wav"))
    else:
        files = [o["inputfile"]]
    devices = o["devices"] or [0]
    if len(files) == 1 and len(devices) > 1:
        # a single recording and several GPUs: split the recording (run() with a device list), not the file list
        return [run_one(files[0], o["outdir"], o["model"], o["frame_size"], o["window"], devices, 0, False)]
    return run_many(files, o["outdir"], o["model"], o["frame_size"], o["window"], devices, o["batch_clips"], run_one)


def run_many(files, outdir, model, frame_size, window, devices, batch_clips, run_one):
    """The reference's only multi-clip driver spawns one Python process per file (separate_multiple.ipynb cell 3); here the
    clips go, longest first, to `len(devices) x batch_clips` resident pipelines (one context / stream each)."""
    import queue
    import threading
    order = sorted(files, key=lambda f: -os.path.getsize(f))
    q = queue.Queue()
    for f in order:
        q.put(f)
    results, errors = {}, []

    def worker(device, slot):
        import torch
        torch.cuda.set_device(device)
        with torch.cuda.stream(torch.cuda.Stream(device=device)):
            while True:
                try:
                    f = q.get_nowait()
                except queue.Empty:
                    return
                try:
                    results[f] = run_one(f, outdir, model, frame_size, window, device, slot, len(files) > 1)
                except Exception as e:  # noqa: BLE001  (reported after the pool drains)
                    errors.append((f, e))
    ths = [threading.Thread(target=worker, args=(d, s)) for d in devices for s in range(batch_clips)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    if errors:
        raise errors[0][1]
    return [results[f] for f in files]
