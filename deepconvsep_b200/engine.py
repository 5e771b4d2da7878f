"""Host side of the H100 separation path: thin Python over the C ABI (libdcs.so).

`Stft` mirrors transform.transformFFT's numerical core, `Separator` mirrors `train_auto` of the
stand-alone scripts (examples/dsd100/separate_dsd.py:239-313).  torch is used only as a
device-memory / stream container; numpy arrays go through the *_host entry points."""
import ctypes as C
import math
from collections import namedtuple
from functools import partial
import numpy as np

from . import _lib
from .models import infer_arch, check_1x1_geometry, gate_code_layout, FAMILY_DEFAULTS


def get_window(window, n):
    """np.hanning / scipy blackmanharris (symmetric) / sinebell by name, callable or array."""
    if isinstance(window, str):
        if window in ("hanning", "hann"):
            return np.hanning(n)
        if window == "blackmanharris":
            from scipy.signal import windows
            return windows.blackmanharris(n)
        if window == "sinebell":
            return np.sin((np.pi * (np.arange(n))) / (1.0 * n))
        raise ValueError("unknown window %r" % window)
    if callable(window):
        return np.asarray(window(n), dtype=np.float64)
    w = np.asarray(window, dtype=np.float64)
    if w.size != n:
        raise ValueError("window has %d samples, frame size is %d" % (w.size, n))
    return w


def _ptr(a):
    """Raw address of a numpy array / torch tensor / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()


def _stream_ptr(stream=None, device=None):
    """cudaStream_t of `stream`, or of torch's current stream ON `device` (the ctx's device: the
    current stream of another device would be a handle the library cannot launch on)."""
    import torch
    s = stream if stream is not None else torch.cuda.current_stream(device)
    return C.c_void_p(s.cuda_stream)


def wiener_stereo(ctx, X, S, iterations, stream=None, num_bins=None, radius=0):
    """Multichannel Wiener post-filter with EM spatial covariances (dcs_wiener_stereo_windowed), in place on device
    spectra: X torch complex64 cuda [2, T, ldf] (the mixture's channels), S [nsrc * 2, T, ldf] (the stems, planes
    ordered (source, channel), nsrc <= 4).  Bins >= num_bins (default ldf) are left alone.  radius: 0 = one spatial
    covariance per source for the whole clip; W >= 1 = per chunk of _lib.WIENER_CHUNK_FRAMES frames, from the chunks
    within W of it.  Returns S."""
    import torch
    if X.dim() != 3 or X.shape[0] != 2 or S.dim() != 3 or S.shape[0] % 2 or tuple(S.shape[1:]) != tuple(X.shape[1:]):
        raise ValueError("wiener_stereo needs X [2, T, ldf] and S [nsrc * 2, T, ldf], got %r and %r"
                         % (tuple(X.shape), tuple(S.shape)))
    if X.dtype != torch.complex64 or S.dtype != torch.complex64 or not (X.is_cuda and S.is_cuda):
        raise ValueError("wiener_stereo needs complex64 cuda tensors")
    if X.stride(2) != 1 or X.stride(1) != X.shape[2] or S.stride(2) != 1 or S.stride(1) != S.shape[2]:
        raise ValueError("wiener_stereo needs contiguous [T, ldf] planes")
    T, ldf = int(X.shape[1]), int(X.shape[2])
    F = ldf if num_bins is None else int(num_bins)
    _lib.check(ctx.lib.dcs_wiener_stereo_windowed(ctx.handle, _ptr(X), X.stride(0), _ptr(S), S.stride(0), S.shape[0] // 2, T,
                                                  ldf, F, int(iterations), int(radius), _stream_ptr(stream, ctx.device)))
    return S


# the channel counts the C-channel Wiener post-filter serves (dcs_wiener_channels): one channel has no spatial covariance
WIENER_CHANNELS = (2, 8)


def check_wiener_channels(nx):
    """ValueError unless the Wiener post-filter serves `nx` channels."""
    lo, hi = WIENER_CHANNELS
    if not lo <= nx <= hi:
        raise ValueError("the Wiener post-filter works on %d to %d channels (one channel has no spatial covariance), got %d"
                         % (lo, hi, nx))


def wiener_channels(ctx, X, S, iterations, stream=None, num_bins=None, radius=0):
    """The multichannel Wiener post-filter on nx = 2 .. 8 channels (dcs_wiener_channels), in place on device spectra:
    X torch complex64 cuda [nx, T, ldf] (the mixture's channels), S [nsrc * nx, T, ldf] (the stems, planes ordered
    (source, channel), nsrc <= 4).  At nx = 2 the bytes of wiener_stereo.  Bins >= num_bins (default ldf) are left
    alone; radius as in wiener_stereo.  Returns S."""
    import torch
    if X.dim() != 3 or S.dim() != 3 or tuple(S.shape[1:]) != tuple(X.shape[1:]) or S.shape[0] % max(X.shape[0], 1):
        raise ValueError("wiener_channels needs X [nx, T, ldf] and S [nsrc * nx, T, ldf], got %r and %r"
                         % (tuple(X.shape), tuple(S.shape)))
    nx = int(X.shape[0])
    check_wiener_channels(nx)
    if X.dtype != torch.complex64 or S.dtype != torch.complex64 or not (X.is_cuda and S.is_cuda):
        raise ValueError("wiener_channels needs complex64 cuda tensors")
    if X.stride(2) != 1 or X.stride(1) != X.shape[2] or S.stride(2) != 1 or S.stride(1) != S.shape[2]:
        raise ValueError("wiener_channels needs contiguous [T, ldf] planes")
    T, ldf = int(X.shape[1]), int(X.shape[2])
    F = ldf if num_bins is None else int(num_bins)
    _lib.check(ctx.lib.dcs_wiener_channels(ctx.handle, _ptr(X), nx, X.stride(0), _ptr(S), S.stride(0), S.shape[0] // nx, T,
                                           ldf, F, int(iterations), int(radius), _stream_ptr(stream, ctx.device)))
    return S


# the networks whose input is not one magnitude plane: their masks cannot come from a downmix inside the library
MASKS_BY_HAND = ("dsd_ild", "bach10_score", "bach10_score_1x1")


def check_channels_family(family):
    """Separator.separate_channels (the downmix's masks applied to every channel) serves the single-channel networks;
    raises ValueError naming the alternative for the others."""
    if family in MASKS_BY_HAND:
        raise ValueError("the %s network does not take a downmix: get its masks with Separator.separate_masks and apply "
                         "them to the channels with Separator.apply_masks" % (family,))


def check_stereo_options(family, keep_channels=False, wiener=0, wiener_radius=0, channels=None):
    """The rule for the options of two-channel stems, by network family (the keys of models.FAMILY_DEFAULTS, which
    are also the Separator's architecture names): keep_channels (the soft masks of the downmix applied to each
    channel) exists for the DSD100 / hiphopss network "dsd" only; wiener (EM iterations of the multichannel Wiener
    post-filter) cannot be negative and needs two-channel stems: keep_channels, or the stereo / ILD network
    "dsd_ild"; wiener_radius (the filter's covariance window in chunks to either side, 0 = the whole clip) cannot be
    negative and needs wiener > 0.  channels: the recording's channel count where it is known and keep_channels is
    asked for -- None or 2 is the rule above; 1 is refused; C > 2 (5.1, arrays: Separator.separate_channels) is served
    for every single-channel network, without the Wiener filter here: the filtered C-channel stems (C <= 8) are
    Separator.separate_channels(wiener=K), which the command-line options do not reach yet.  Raises ValueError with the
    reason otherwise."""
    if keep_channels and channels is not None and channels != 2:
        if channels < 2:
            raise ValueError("--keep-channels needs at least a 2-channel recording, this one has %d channel(s)" % channels)
        check_channels_family(family)
        if wiener:
            raise ValueError("--wiener %d: the Wiener post-filter works on two-channel stems, this recording has %d "
                             "channels" % (wiener, channels))
        return check_wiener_radius(wiener, wiener_radius)
    if keep_channels and family != "dsd":
        raise ValueError("--keep-channels: only the DSD100 / hiphopss network (family dsd) keeps the stereo channels, "
                         "not %s" % (family,))
    if wiener < 0:
        raise ValueError("--wiener %d: the number of EM iterations cannot be negative" % wiener)
    if wiener and not (keep_channels or family == "dsd_ild"):
        raise ValueError("--wiener needs --keep-channels (family dsd) or the stereo / ILD network (family dsd_ild): "
                         "the Wiener post-filter works on two-channel stems")
    check_wiener_radius(wiener, wiener_radius)


def check_wiener_radius(wiener, wiener_radius):
    """The wiener_radius half of check_stereo_options, for the calls whose network and layout are already fixed."""
    if wiener_radius < 0:
        raise ValueError("--wiener-radius %d: the covariance window cannot be negative" % wiener_radius)
    if wiener_radius and not wiener:
        raise ValueError("--wiener-radius needs --wiener K > 0: it is the window of the Wiener post-filter's covariances")


def clip_call(sep, filters=None, melody=None, frame0=0, keep_channels=False, wiener=0, wiener_radius=0, channels=None):
    """The call that separates a whole clip with Separator `sep`'s network and these inputs, as a function of the
    audio: sep.separate_channels (keep_channels=True on a recording of `channels` > 2 channels),
    sep.separate_keep_channels (keep_channels=True otherwise), sep.separate_notes (the note table melody, from table frame
    frame0), sep.separate_score (a score-informed net and its score filters), sep.separate_stereo (the stereo / ILD
    net) or sep.separate.  wiener: EM iterations of the Wiener post-filter, and wiener_radius its covariance window
    (passed only when set), given to the two-channel calls and refused for the others here, before anything runs.
    Only sep.model.arch and the method picked are used, so stand-ins with just those work too."""
    rkw = {"wiener_radius": wiener_radius} if wiener_radius else {}
    if keep_channels and channels is not None and channels != 2:
        check_stereo_options(sep.model.arch, True, wiener, wiener_radius, channels)
        return sep.separate_channels
    if keep_channels:
        return partial(sep.separate_keep_channels, wiener=wiener, **rkw)
    if melody is not None:
        run = partial(sep.separate_notes, melody=melody, frame0=frame0)
    elif sep.model.arch in ("bach10_score", "bach10_score_1x1"):
        run = partial(sep.separate_score, filters=filters)
    elif sep.model.arch == "dsd_ild":
        return partial(sep.separate_stereo, wiener=wiener, **rkw)
    else:
        run = sep.separate
    check_stereo_options(sep.model.arch, wiener=wiener, wiener_radius=wiener_radius)
    return run


def check_melody(melody, ninst=None):
    """The note table (deepconvsep_b200.score.score_melody) as the library takes it: float64 C-contiguous
    [ninst, nnotes, ncols], ninst in 1..4 (`ninst` when given), ncols >= 3.  The rows themselves are checked by the
    library before it queues anything (include/dcs.h, dcs_score_filters)."""
    m = np.ascontiguousarray(melody, dtype=np.float64)
    if m.ndim != 3:
        raise ValueError("melody must be [ninst, nnotes, ncols], got shape %r" % (m.shape,))
    if not 1 <= m.shape[0] <= 4 or (ninst is not None and m.shape[0] != ninst):
        raise ValueError("melody has %d instruments, %s" % (m.shape[0], "the model takes %d" % ninst if ninst else "1 to 4 allowed"))
    if m.shape[2] < 3:
        raise ValueError("melody rows have %d columns, at least 3 (first frame, last frame, MIDI number)" % m.shape[2])
    return m


def score_filters(ctx, melody, T, F, start=0, mag=None, ldf=None, stream=None):
    """filterSpec(mag, melody, start, start + T) rasterised on the device (dcs_score_filters) -> torch float32 cuda
    [ninst, T, ldf], pad columns 0.  mag None: the normalised filters; mag (torch float32 cuda [T, ldf]): the filters
    times mag.  ldf defaults to mag's row length, else F rounded up to 8."""
    import torch
    m = check_melody(melody)
    T, F, start = int(T), int(F), int(start)
    if T < 1 or F < 1 or start < 0:
        raise ValueError("score_filters: T %d and F %d must be >= 1, start %d >= 0" % (T, F, start))
    if mag is not None:
        if not (mag.is_cuda and mag.dtype == torch.float32 and mag.dim() == 2 and mag.shape[0] == T and mag.is_contiguous()):
            raise ValueError("mag must be a contiguous float32 cuda tensor [T, ldf]")
        ldf = mag.shape[1] if ldf is None else ldf
        if mag.shape[1] != ldf:
            raise ValueError("mag has rows of %d, ldf is %d" % (mag.shape[1], ldf))
    ldf = int(ldf if ldf is not None else (F + 7) // 8 * 8)
    out = torch.empty((m.shape[0], T, ldf), dtype=torch.float32, device=torch.device("cuda", ctx.device))
    _lib.check(ctx.lib.dcs_score_filters(ctx.handle, m.ctypes.data, m.shape[0], m.shape[1], m.shape[2], start, T, F,
                                         _ptr(mag), ldf, _ptr(out), T * ldf, _stream_ptr(stream, ctx.device)))
    return out


# every network was trained on spectra of 44.1 kHz audio; other rates go through a Resampler
MODEL_RATE = 44100
# packed signed 24-bit little-endian PCM, 3 bytes per sample: a clip [L, C] of it is what
# np.memmap(path, dtype=PCM24, offset=data_offset, shape=(L, C)) gives for the data chunk of a 24-bit WAV
PCM24 = np.dtype("V3")
# the sample formats of separate_channels_batch: numpy dtype -> DCS_SAMPLE_* (include/dcs.h)
_SAMPLE_FORMATS = {np.dtype(np.int16): _lib.SAMPLE_I16, np.dtype(np.int32): _lib.SAMPLE_I32,
                   np.dtype(np.float32): _lib.SAMPLE_F32, PCM24: _lib.SAMPLE_I24}
# the sample rates a Resampler takes: integers in this range whose polyphase bank fits, in both directions
RESAMPLE_RATES = (8000, 192000)
# one segment of Separator.long_segments: the recording's samples staged, the range separated at 44.1 kHz, the core kept
LongSegment = namedtuple("LongSegment", "in_start in_stop model_start model_stop out_start out_stop")


def resample_ratio(rate_in, rate_out):
    """(up, down): rate_out / rate_in in lowest terms."""
    from math import gcd
    g = gcd(int(rate_in), int(rate_out))
    return int(rate_out) // g, int(rate_in) // g


def resample_taps(up, down):
    """The filter scipy.signal.resample_poly(x, up, down) designs by default, float64 [20 * max(up, down) + 1]:
    firwin(2 * half_len + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, half_len = 10 * max(up, down)."""
    from scipy.signal import firwin
    m = max(int(up), int(down))
    return np.ascontiguousarray(firwin(2 * 10 * m + 1, 1.0 / m, window=("kaiser", 5.0)) * int(up), dtype=np.float64)


def resample_bank_bytes(up, down):
    """Bytes of the polyphase bank of resample_taps(up, down): ceil(ntaps / up) taps for each of the up phases."""
    ntaps = 20 * max(up, down) + 1
    return -(-ntaps // up) * up * 8


def check_resample_rates(rate_in, rate_out):
    """(up, down) for resampling rate_in -> rate_out; ValueError naming the rate unless both are integers in
    RESAMPLE_RATES whose bank is at most _lib.RESAMPLE_MAX_BANK_BYTES in both directions."""
    lo, hi = RESAMPLE_RATES
    for r in (rate_in, rate_out):
        if isinstance(r, bool) or not isinstance(r, (int, float, np.integer, np.floating)) or r != int(r):
            raise ValueError("sample rate %r Hz: only integer rates are resampled" % (r,))
        if not lo <= int(r) <= hi:
            raise ValueError("sample rate %d Hz: rates from %d to %d Hz are resampled" % (int(r), lo, hi))
    up, down = resample_ratio(rate_in, rate_out)
    worst = max(resample_bank_bytes(up, down), resample_bank_bytes(down, up))
    if worst > _lib.RESAMPLE_MAX_BANK_BYTES:
        odd = int(rate_in) if int(rate_out) == MODEL_RATE else int(rate_out)
        raise ValueError("sample rate %d Hz: %d <-> %d Hz reduces to %d/%d, whose polyphase filter bank (%d bytes) is over "
                         "the %d a resampler takes; resample it to a nearby common rate first"
                         % (odd, int(rate_in), int(rate_out), up, down, worst, _lib.RESAMPLE_MAX_BANK_BYTES))
    return up, down


class Resampler(object):
    """rate_in -> rate_out on the device (dcs_resample): scipy.signal.resample_poly with its default filter and zero
    padding, the taps in fp64, rounded once to fp32.  Rates as check_resample_rates accepts them."""

    def __init__(self, ctx, rate_in, rate_out):
        self.up, self.down = check_resample_rates(rate_in, rate_out)
        self.rate_in, self.rate_out = int(rate_in), int(rate_out)
        self.ctx, self.lib = ctx, ctx.lib
        self.taps = resample_taps(self.up, self.down)
        h = C.c_void_p()
        _lib.check(self.lib.dcs_resampler_create(ctx.handle, self.up, self.down, self.taps.ctypes.data, self.taps.size,
                                                 C.byref(h)))
        self.handle = h

    def length(self, num_in):
        """ceil(num_in * up / down): the samples of the whole resampled signal"""
        return int(self.lib.dcs_resampled_length(int(num_in), self.up, self.down))

    def resample(self, planes, num_out=None, stream=None, out=None):
        """planes: float32 cuda [P, L] (rows contiguous, gaps between planes allowed) -> float32 cuda [P, num_out]
        (default self.length(L); shorter trims the tail), into `out` when given ([P, num_out], rows contiguous)."""
        import torch
        if planes.dim() != 2 or planes.dtype != torch.float32 or not planes.is_cuda or planes.stride(1) != 1:
            raise ValueError("resample needs float32 cuda planes [P, L] with contiguous rows, got %r %s"
                             % (tuple(planes.shape), planes.dtype))
        P, L = planes.shape
        n = self.length(L) if num_out is None else int(num_out)
        if out is None:
            out = torch.empty((P, n), dtype=torch.float32, device=planes.device)
        elif not (out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (P, n) and out.stride(1) == 1):
            raise ValueError("resample: out must be float32 cuda [%d, %d] with contiguous rows" % (P, n))
        _lib.check(self.lib.dcs_resample(self.handle, _ptr(planes), P, planes.stride(0), L, _ptr(out), out.stride(0), n,
                                         _stream_ptr(stream, self.ctx.device)))
        return out

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dcs_resampler_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_SCORE_AT_RATE = "resample the audio to 44.1 kHz with Resampler first, and give the score on that grid"
_MASKS_AT_RATE = ("resample the audio to 44.1 kHz with Resampler first, or use separate / separate_channels with "
                  "sample_rate=, which resample for you")


def check_model_rate(sample_rate, call, alternative):
    """ValueError unless sample_rate is the networks' 44.1 kHz, for the calls whose inputs are on its grids."""
    if sample_rate != MODEL_RATE:
        raise ValueError("%s works at %d Hz only (sample_rate %r): %s" % (call, MODEL_RATE, sample_rate, alternative))


class Context(object):
    """One dcs_ctx = one device + the workspace of one in-flight pipeline."""

    def __init__(self, device=0):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.dcs_create(int(device), C.byref(h)))
        self.handle = h
        self.device = int(device)

    def launch_count(self):
        return int(self.lib.dcs_launch_count(self.handle))

    def workspace_bytes(self):
        return int(self.lib.dcs_workspace_bytes(self.handle))

    def profile(self, enable):
        _lib.check(self.lib.dcs_profile(self.handle, 1 if enable else 0))

    def set_wiener(self, iterations):
        """EM iterations of the Wiener post-filter on the context's two-channel stems (dcs_set_wiener; 0 = off)"""
        _lib.check(self.lib.dcs_set_wiener(self.handle, int(iterations)))

    def set_wiener_radius(self, radius):
        """covariance window of that filter in chunks of _lib.WIENER_CHUNK_FRAMES frames to either side
        (dcs_set_wiener_radius; 0 = the whole clip)"""
        _lib.check(self.lib.dcs_set_wiener_radius(self.handle, int(radius)))

    def profile_read(self, max_n=4096):
        """[(stage name, milliseconds)] recorded since profiling was enabled (synchronises)."""
        names = C.create_string_buffer(64 * max_n)
        ms = (C.c_float * max_n)()
        n = self.lib.dcs_profile_read(self.handle, names, len(names), ms, max_n)
        if n < 0:
            _lib.check(n)
        nm = names.value.decode().split("\n")[:n]
        return list(zip(nm, [float(ms[i]) for i in range(n)]))

    def gemm(self, A, B, bias=None, relu=False, engine=1, stream=None):
        """torch float32 cuda A [M,K] (row stride A.stride(0)) x numpy B [K,N] -> torch [M,N]."""
        import torch
        M, K = A.shape
        Bh = np.ascontiguousarray(B, dtype=np.float32)
        N = Bh.shape[1]
        bh = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
        Cd = torch.empty((M, N), dtype=torch.float32, device=A.device)
        _lib.check(self.lib.dcs_gemm_f32(self.handle, int(engine), _ptr(A), A.stride(0), Bh.ctypes.data, N,
                                         None if bh is None else bh.ctypes.data, _ptr(Cd), N, M, N, K, int(relu),
                                         _stream_ptr(stream, self.device)))
        return Cd

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dcs_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Stft(object):
    """STFT plan (frame size, hop, analysis/synthesis windows)."""

    def __init__(self, ctx, frame_size, hop, window=np.hanning, syn_window=None):
        self.ctx, self.lib = ctx, ctx.lib
        self.N, self.hop = int(frame_size), int(hop)
        self.device = ctx.device
        self.F = self.N // 2 + 1
        self.ldf = int(self.lib.dcs_padded_bins(self.N))
        self.window = np.ascontiguousarray(get_window(window, self.N), dtype=np.float64)
        syn = None if syn_window is None else np.ascontiguousarray(get_window(syn_window, self.N), dtype=np.float64)
        h = C.c_void_p()
        _lib.check(self.lib.dcs_stft_plan(ctx.handle, self.N, self.hop, self.window.ctypes.data,
                                          None if syn is None else syn.ctypes.data, C.byref(h)))
        self.handle = h

    @property
    def dev(self):
        import torch
        return torch.device("cuda", self.device)

    def num_frames(self, L):
        return int(self.lib.dcs_num_frames(int(L), self.hop))

    def out_length(self, T):
        return (T - 1) * self.hop + self.N - self.N // 2

    # ---- device-tensor API (torch) ----
    def forward(self, audio, mag_scale=1.0, want_X=True, want_mag=True, stream=None):
        """audio: torch float32 cuda [L] -> (X complex64 [T, ldf] | None, mag float32 [T, ldf] | None)"""
        import torch
        L = audio.numel()
        T = self.num_frames(L)
        X = torch.empty((T, self.ldf), dtype=torch.complex64, device=audio.device) if want_X else None
        mag = torch.empty((T, self.ldf), dtype=torch.float32, device=audio.device) if want_mag else None
        _lib.check(self.lib.dcs_stft_forward(self.handle, _ptr(audio), L, _ptr(X), _ptr(mag), float(mag_scale),
                                             self.ldf, _stream_ptr(stream, self.device)))
        return X, mag

    def forward_polar(self, audio, mag_scale=1.0, stream=None):
        import torch
        L = audio.numel()
        T = self.num_frames(L)
        mag = torch.empty((T, self.ldf), dtype=torch.float32, device=audio.device)
        ph = torch.empty((T, self.ldf), dtype=torch.float32, device=audio.device)
        _lib.check(self.lib.dcs_stft_forward_polar(self.handle, _ptr(audio), L, _ptr(mag), _ptr(ph), float(mag_scale),
                                                   self.ldf, _stream_ptr(stream, self.device)))
        return mag, ph

    def inverse(self, S, num_out=None, stream=None):
        """S: torch complex64 cuda [nsrc, T, ldf] (or [T, ldf]) -> float32 [nsrc, num_out]"""
        import torch
        if S.dim() == 2:
            S = S.unsqueeze(0)
        nsrc, T, ldf = S.shape
        assert S.is_contiguous() and ldf >= self.F
        n = self.out_length(T) if num_out is None else int(num_out)
        out = torch.empty((nsrc, n), dtype=torch.float32, device=S.device)
        _lib.check(self.lib.dcs_istft(self.handle, _ptr(S), nsrc, T, ldf, T * ldf, _ptr(out), n, n, _stream_ptr(stream, self.device)))
        return out

    def inverse_masked(self, X, M, num_out=None, stream=None):
        """istft_norm(M_s * X_c) with the product formed inside the kernel (dcs_istft_masked): X torch complex64 cuda
        [nx, T, ldf] (or [T, ldf]), M float32 cuda [nsrc, T, ldf] (or [T, ldf]) with rows of the same ldf -> float32
        [nsrc * nx, num_out], plane (s * nx + c).  The planes may be views with gaps between them; rows are contiguous."""
        import torch
        X = X.unsqueeze(0) if X.dim() == 2 else X
        M = M.unsqueeze(0) if M.dim() == 2 else M
        if X.dim() != 3 or M.dim() != 3 or tuple(X.shape[1:]) != tuple(M.shape[1:]):
            raise ValueError("inverse_masked needs X [nx, T, ldf] and M [nsrc, T, ldf], got %r and %r" % (tuple(X.shape), tuple(M.shape)))
        if X.dtype != torch.complex64 or M.dtype != torch.float32 or not (X.is_cuda and M.is_cuda):
            raise ValueError("inverse_masked needs a complex64 X and a float32 M on the device")
        nx, T, ldf = X.shape
        if any(t.stride(2) != 1 or t.stride(1) != ldf for t in (X, M)) or ldf < self.F:
            raise ValueError("inverse_masked needs contiguous rows of ldf >= %d" % self.F)
        n = self.out_length(T) if num_out is None else int(num_out)
        out = torch.empty((M.shape[0] * nx, n), dtype=torch.float32, device=X.device)
        _lib.check(self.lib.dcs_istft_masked(self.handle, _ptr(X), nx, X.stride(0), _ptr(M), M.shape[0], M.stride(0), T, ldf,
                                             _ptr(out), n, n, _stream_ptr(stream, self.device)))
        return out

    def inverse_polar(self, mag, phase, mag_scale=1.0, num_out=None, stream=None):
        import torch
        T, ldf = mag.shape
        n = self.out_length(T) if num_out is None else int(num_out)
        out = torch.empty((n,), dtype=torch.float32, device=mag.device)
        _lib.check(self.lib.dcs_istft_polar(self.handle, self.ctx.handle, _ptr(mag), _ptr(phase), float(mag_scale), T, ldf,
                                            _ptr(out), n, _stream_ptr(stream, self.device)))
        return out

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dcs_stft_plan_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Model(object):
    """Device-resident network built from a Lasagne parameter list."""

    def __init__(self, ctx, params, arch=None, feat_size=None, time_context=None):
        self.ctx, self.lib = ctx, ctx.lib
        try:
            ia, iF, itc = infer_arch(params, feat_size)   # time_context None: the one the weights were trained with
        except ValueError:
            if arch is None or feat_size is None:
                raise
            ia, iF, itc = arch, feat_size, 30
        a = ia if arch is None else arch
        F = feat_size if (arch is not None and feat_size is not None) else iF
        self.arch, self.F, self.tc = a, int(F), int(time_context or itc)
        if a == "bach10_score_1x1":
            check_1x1_geometry(self.F, self.tc)
        arrs = [np.ascontiguousarray(p, dtype=np.float32) for p in params]
        n = len(arrs)
        ptrs = (C.c_void_p * n)(*[x.ctypes.data for x in arrs])
        shapes = np.ones((n, 4), dtype=np.int64)
        ndims = np.zeros(n, dtype=np.int32)
        for i, x in enumerate(arrs):
            ndims[i] = x.ndim
            shapes[i, :x.ndim] = x.shape
        h = C.c_void_p()
        _lib.check(self.lib.dcs_model_create(ctx.handle, _lib.ARCH_IDS[a], self.F, self.tc, n, ptrs,
                                             shapes.ctypes.data, ndims.ctypes.data, C.byref(h)))
        self.handle = h
        self.nsrc = int(self.lib.dcs_model_nsources(h))

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dcs_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Separator(object):
    """train_auto() as an object: build once (weights uploaded, plan made), call many times."""

    def __init__(self, params, arch=None, frame_size=None, hop=None, window=None, scale_factor=0.3,
                 time_context=None, overlap=None, patcher="standalone", device=0, feat_size=None):
        self.ctx = Context(device)
        if arch is None and frame_size is not None and feat_size is None:
            feat_size = frame_size // 2 + 1
        self.model = Model(self.ctx, params, arch=arch, feat_size=feat_size, time_context=time_context)
        d = FAMILY_DEFAULTS[self.model.arch]
        self.frame_size = int(frame_size or 2 * (self.model.F - 1))
        self.hop = int(hop or d["hopSize"])
        self.window = window if window is not None else d["window"]
        self.overlap = int(d["overlap"] if overlap is None else overlap)
        self.scale_factor = float(scale_factor)
        self.patcher = _lib.PATCHER_IDS[patcher]
        self.stft = Stft(self.ctx, self.frame_size, self.hop, self.window)
        self.nsrc = self.model.nsrc
        self.sources = d["sources"]
        self.lib = self.ctx.lib
        self._resamplers = {}

    def resampler(self, rate_in, rate_out):
        """The Resampler rate_in -> rate_out on this separator's context, made on first use and kept."""
        key = (rate_in, rate_out)
        if key not in self._resamplers:
            self._resamplers[key] = Resampler(self.ctx, rate_in, rate_out)
        return self._resamplers[key]

    def _at_rate(self, call, audio, sample_rate, out, stream, channels=None, mono=False):
        """A stems call on audio at sample_rate != MODEL_RATE: the audio planes to MODEL_RATE, call(planes, stream=stream)
        on them (the device entry point), the nsrc x C stem planes back in one launch, trimmed to the input's length.
        audio as the channel calls take it with `channels` (None: 1 to 16), or mono float [L] (numpy or cuda tensor)
        -> the layout of the call at MODEL_RATE: numpy [nsrc, L] (mono) or [L, nsrc, C], or device planes [nsrc * C, L]."""
        down = self.resampler(sample_rate, MODEL_RATE)     # the rate is checked before any device work
        back = self.resampler(MODEL_RATE, sample_rate)
        if mono:
            import torch
            host = not hasattr(audio, "is_cuda")
            x = torch.as_tensor(np.ascontiguousarray(audio, dtype=np.float32), device=self.stft.dev) if host else audio
            if x.dim() != 1 or x.dtype != torch.float32:
                raise ValueError("this network needs mono float audio [L], got %r" % (tuple(x.shape),))
            x = x.contiguous().unsqueeze(0)
            outd = out if (out is not None and not host) else None
            stems = back.resample(call(down.resample(x, stream=stream)[0], stream=stream), num_out=x.shape[1],
                                  stream=stream, out=outd)
            if not host:
                return stems
            if out is not None:
                out[...] = stems.cpu().numpy()
                return out
            return stems.cpu().numpy()
        host, x, outd = self._channel_planes(audio, out, self.nsrc, channels)
        back.resample(call(down.resample(x, stream=stream), stream=stream), num_out=x.shape[1], stream=stream, out=outd)
        return self._channel_stems(host, outd, out, x.shape[0])

    # ---- host buffers (numpy): H2D + pipeline + D2H inside the call ----
    def separate(self, audio, out=None, sample_rate=MODEL_RATE):
        """audio: 1-D float array (any float dtype) -> float32 [nsrc, L].  `audio` / `out` may be
        pinned (torch.from_numpy(...).pin_memory() views) for asynchronous copies.
        sample_rate: the audio's rate.  At MODEL_RATE (44.1 kHz) this call; at another rate (check_resample_rates) the
        audio is resampled to 44.1 kHz on the device, separated there (separate_device) and the stems resampled back to
        the input's rate and length -- a float32 cuda tensor [L] in then gives the device stems [nsrc, L]."""
        if sample_rate != MODEL_RATE:
            return self._at_rate(self.separate_device, audio, sample_rate, out, None, mono=True)
        a = np.ascontiguousarray(audio, dtype=np.float32)
        L = a.size
        if out is None:
            out = np.empty((self.nsrc, L), dtype=np.float32)
        assert out.dtype == np.float32 and out.shape == (self.nsrc, L) and out.flags.c_contiguous
        _lib.check(self.lib.dcs_separate_host(self.ctx.handle, self.model.handle, self.stft.handle, a.ctypes.data, L,
                                              self.scale_factor, self.overlap, self.patcher, out.ctypes.data, L,
                                              _stream_ptr(None, self.ctx.device)))
        return out

    def separate_pcm16(self, pcm, downmix=1, out=None, keep_channels=False, wiener=0, wiener_radius=0):
        """int16 wav samples [L] or [L, channels] -> int16 [nsrc, L] (train_auto's wav contract).
        keep_channels=True (DSD100 / hiphopss net, stereo [L, 2] in): int16 [nsrc, L, 2] stereo stems, see
        separate_keep_channels; wiener: EM iterations of the Wiener post-filter on them and wiener_radius its
        covariance window (keep_channels only)."""
        if keep_channels:
            return self.separate_pcm16_batch([pcm], outs=None if out is None else [out], keep_channels=True,
                                             wiener=wiener, wiener_radius=wiener_radius)[0]
        check_stereo_options(self.model.arch, wiener=wiener, wiener_radius=wiener_radius)
        p = np.ascontiguousarray(pcm, dtype=np.int16)
        L = p.shape[0]
        ch = 1 if p.ndim == 1 else p.shape[1]
        if out is None:
            out = np.empty((self.nsrc, L), dtype=np.int16)
        _lib.check(self.lib.dcs_separate_pcm16_host(self.ctx.handle, self.model.handle, self.stft.handle, p.ctypes.data, L,
                                                    ch, int(downmix if ch > 1 else 0), self.scale_factor, self.overlap,
                                                    self.patcher, out.ctypes.data, L, _stream_ptr(None, self.ctx.device)))
        return out

    def separate_pcm16_batch(self, clips, downmix=1, outs=None, keep_channels=False, wiener=0, wiener_radius=0):
        """Several clips through the context's multi-clip scheduler (dcs_separate_batch_pcm16_host): H2D of clip i+1,
        the kernels of clip i and D2H of clip i-1 overlap.  clips: list of int16 arrays [L] or [L, channels] (same
        channel count; pinned for real overlap) -> list of int16 [nsrc, L].  keep_channels=True: stereo clips
        [L, 2] -> list of int16 [nsrc, L, 2] (dcs_separate_batch_pcm16_keep_channels_host), with `wiener` EM iterations
        of the Wiener post-filter on each clip's stems, over covariance windows of `wiener_radius` chunks."""
        if not keep_channels:
            check_stereo_options(self.model.arch, wiener=wiener, wiener_radius=wiener_radius)
        ps = [np.ascontiguousarray(c, dtype=np.int16) for c in clips]
        if not ps:
            return []
        if keep_channels:
            for p_ in ps:
                if p_.ndim != 2 or p_.shape[1] != 2:
                    raise ValueError("keep_channels needs stereo int16 clips [L, 2], got shape %r" % (p_.shape,))
            check_wiener_radius(wiener, wiener_radius)
            self.ctx.set_wiener(wiener)
            self.ctx.set_wiener_radius(wiener_radius)
            return self._pcm16_batch(self.lib.dcs_separate_batch_pcm16_keep_channels_host, ps, outs, (2,), ())
        ch = 1 if ps[0].ndim == 1 else ps[0].shape[1]
        assert all((1 if p_.ndim == 1 else p_.shape[1]) == ch for p_ in ps), "all clips must have the same channel count"
        return self._pcm16_batch(self.lib.dcs_separate_batch_pcm16_host, ps, outs, (), (ch, int(downmix if ch > 1 else 0)))

    def separate_pcm16_channels_batch(self, clips, outs=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE):
        """C-channel int16 clips through the context's multi-clip scheduler (dcs_separate_batch_pcm16_channels_host):
        H2D of clip i+1, the kernels of clip i and D2H of clip i-1 overlap, and the decode to fp32 and the encode of the
        stems to int16 run on the device.  clips: list of int16 arrays [L, C] with the same C in 1..16 (pinned for real
        overlap) -> list of int16 [nsrc, L, C] (into `outs` when given, which may be pinned): per clip
        (separate_channels(clip / 32767, wiener, wiener_radius, sample_rate) * 32767) truncated to int16 in fp32, source
        by source.  wiener > 0 (C in 2..8): EM iterations of the Wiener post-filter, over covariance windows of
        wiener_radius chunks.  At C = 2 with the DSD100 network, the bytes of separate_pcm16_batch(keep_channels=True)
        with the same wiener and wiener_radius.
        sample_rate: the clips' rate, one for the whole call (a sequence of one rate per clip is taken if they are all
        equal).  At another rate than MODEL_RATE (check_resample_rates) each clip is resampled to 44.1 kHz as it is
        decoded and its stems back to its own rate and length as they are encoded, on the device with this separator's
        resamplers (dcs_separate_batch_pcm16_channels_resampled_host): no more launches per clip than at 44.1 kHz."""
        ps, ch, args, sample_rate = self._channels_clips("separate_pcm16_channels_batch", clips, (np.int16,), wiener,
                                                         wiener_radius, sample_rate)
        if not ps:
            return []
        if sample_rate == MODEL_RATE:
            return self._pcm16_batch(self.lib.dcs_separate_batch_pcm16_channels_host, ps, outs, (ch,), args)
        pre = (self.resampler(sample_rate, MODEL_RATE).handle, self.resampler(MODEL_RATE, sample_rate).handle)
        return self._pcm16_batch(self.lib.dcs_separate_batch_pcm16_channels_resampled_host, ps, outs, (ch,), args, pre)

    def separate_channels_batch(self, clips, outs=None, out_dtype=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE):
        """separate_pcm16_channels_batch for int16, int32 or float32 clips (dcs_separate_batch_channels_host): 24-bit
        PCM as scipy.io.wavfile reads it (int32, the sample in the top 24 bits), 32-bit PCM, or IEEE float.  clips:
        list of arrays [L, C] of one dtype and one C in 1..16 -> list of [nsrc, L, C] arrays of out_dtype (default the
        clips' dtype; int16, int32 or float32), into `outs` when given.  Per clip the stems are
        encode(separate_channels(decode(clip), wiener, wiener_radius, sample_rate)), with the rules of include/dcs.h:
        int16 decodes as clip / 32767 and encodes as (stem * 32767) truncated in fp32, wrapping; int32 decodes as
        (clip / (2^31 - 1)) in fp64 rounded to fp32 and encodes as stem * (2^31 - 1) in fp64, truncated and saturated;
        float32 is taken and given back as it is, without scaling or clipping.  PCM24 (packed 3-byte samples, the bytes of
        a 24-bit WAV data chunk, util.wav_samples) decodes as the int32 rule on the sample shifted left by 8 and encodes
        as the int32 encode shifted right by 8: the same values as int32 for 24-bit material, with a quarter fewer
        bytes over the host link.  The conversions run on the device, fused into the resamplers at another rate.  With
        int16 in and out, the bytes of separate_pcm16_channels_batch."""
        ps, ch, args, sample_rate = self._channels_clips("separate_channels_batch", clips, tuple(_SAMPLE_FORMATS), wiener,
                                                         wiener_radius, sample_rate)
        dtypes = {p_.dtype for p_ in ps}
        if len(dtypes) > 1:
            raise ValueError("all clips of a batch must have the same dtype, got %s" % sorted(str(d) for d in dtypes))
        in_dtype = ps[0].dtype if ps else np.dtype(np.int16)
        try:
            out_dtype = in_dtype if out_dtype is None else np.dtype(out_dtype)
        except TypeError:
            raise ValueError("separate_channels_batch: out_dtype %r is not a dtype" % (out_dtype,))
        if out_dtype not in _SAMPLE_FORMATS:
            raise ValueError("separate_channels_batch encodes int16, int32, float32 or PCM24 (V3) stems, not %s" % out_dtype)
        if not ps:
            return []
        pre = (None, None)
        if sample_rate != MODEL_RATE:
            pre = (self.resampler(sample_rate, MODEL_RATE).handle, self.resampler(MODEL_RATE, sample_rate).handle)
        pre += (_SAMPLE_FORMATS[in_dtype], _SAMPLE_FORMATS[out_dtype])
        return self._pcm16_batch(self.lib.dcs_separate_batch_channels_host, ps, outs, (ch,), args, pre, out_dtype)

    def long_segments(self, num_samples, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE, segment_seconds=120.0):
        """The segments separate_long_channels cuts a recording of num_samples samples into (dcs_long_segments): a list
        of LongSegment (in_start, in_stop, model_start, model_stop, out_start, out_stop) for this separator's geometry,
        the filter's reach wiener * wiener_radius and the rate's resampler pair."""
        check_wiener_radius(wiener, wiener_radius)
        if wiener < 0:
            raise ValueError("wiener %d: the number of EM iterations cannot be negative" % wiener)
        core = self._long_core(segment_seconds, sample_rate)
        if sample_rate != MODEL_RATE:
            up, down = check_resample_rates(sample_rate, MODEL_RATE)
            to_taps = from_taps = len(resample_taps(up, down))     # the same length both ways
        else:
            up = down = to_taps = from_taps = 1
        args = (int(num_samples), core, self.frame_size, self.hop, self.model.tc, self.overlap, int(wiener) * int(wiener_radius),
                up, down, to_taps, from_taps)
        n = int(self.lib.dcs_long_segments(*args, None, 0))
        if n < 0:
            raise ValueError("long_segments: no plan for %d samples in cores of %d" % (int(num_samples), core))
        segs = (_lib.Segment * n)()
        self.lib.dcs_long_segments(*args, segs, n)
        return [LongSegment(s.in_start, s.in_stop, s.model_start, s.model_stop, s.out_start, s.out_stop) for s in segs]

    @staticmethod
    def _long_core(segment_seconds, sample_rate):
        """core_samples of segment_seconds at sample_rate; ValueError unless segment_seconds is a finite number > 0"""
        if isinstance(segment_seconds, bool) or not isinstance(segment_seconds, (int, float, np.integer, np.floating)) \
                or not (math.isfinite(segment_seconds) and segment_seconds > 0):
            raise ValueError("segment_seconds %r must be a finite number > 0" % (segment_seconds,))
        return max(1, int(round(float(segment_seconds) * float(sample_rate))))

    def separate_long_channels(self, recording, out=None, out_dtype=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE,
                               segment_seconds=120.0):
        """One C-channel recording of any length through the multi-clip scheduler with a device workspace bounded by the
        segment length (dcs_separate_long_channels_host): recording [L, C] of int16, int32, float32 or PCM24, C in 1..16 ->
        [nsrc, L, C] of out_dtype (default the recording's dtype), into `out` when given.  The recording is cut into
        cores of segment_seconds (long_segments); each segment is separated with the margins that make its core the
        whole recording's stems (up to the GEMMs' summation order for another patch count), and its core is written
        straight into the result.  The sample rules, rates and filter options are those of separate_channels_batch; the
        Wiener post-filter over more than one segment needs wiener_radius >= 1.  120 s keeps the workspace of a
        6-channel filtered recording near that of a 180 s clip."""
        ps, ch, args, sample_rate = self._channels_clips("separate_long_channels", [recording], tuple(_SAMPLE_FORMATS), wiener,
                                                         wiener_radius, sample_rate)
        core = self._long_core(segment_seconds, sample_rate)
        x = ps[0]
        try:
            out_dtype = x.dtype if out_dtype is None else np.dtype(out_dtype)
        except TypeError:
            raise ValueError("separate_long_channels: out_dtype %r is not a dtype" % (out_dtype,))
        if out_dtype not in _SAMPLE_FORMATS:
            raise ValueError("separate_long_channels encodes int16, int32, float32 or PCM24 (V3) stems, not %s" % out_dtype)
        L = x.shape[0]
        if out is None:
            out = np.empty((self.nsrc, L, ch), dtype=out_dtype)
        elif not (isinstance(out, np.ndarray) and out.dtype == out_dtype and out.shape == (self.nsrc, L, ch)
                  and out.flags.c_contiguous):
            raise ValueError("separate_long_channels: out must be a contiguous %s array [%d, %d, %d]" % (out_dtype, self.nsrc, L, ch))
        pre = (None, None)
        if sample_rate != MODEL_RATE:
            pre = (self.resampler(sample_rate, MODEL_RATE).handle, self.resampler(MODEL_RATE, sample_rate).handle)
        _lib.check(self.lib.dcs_separate_long_channels_host(
            self.ctx.handle, self.model.handle, self.stft.handle, *pre, _SAMPLE_FORMATS[x.dtype], _SAMPLE_FORMATS[out_dtype],
            x.ctypes.data, L, *args, core, self.scale_factor, self.overlap, self.patcher, out.ctypes.data, L,
            _stream_ptr(None, self.ctx.device)))
        return out

    def _channels_clips(self, call, clips, dtypes, wiener, wiener_radius, sample_rate):
        """the checks of the C-channel batch calls, before any library call: the network, the filter options, clips
        [L, C] of one of `dtypes` with one C in 1..16, one sample rate -> (contiguous clips, C, the entry's arguments
        between the clip lengths and scale_factor, the rate)"""
        check_channels_family(self.model.arch)
        check_wiener_radius(wiener, wiener_radius)
        if wiener < 0:
            raise ValueError("wiener %d: the number of EM iterations cannot be negative" % wiener)
        ps = []
        for c in clips:
            a = np.asarray(c)
            if a.dtype not in dtypes or a.ndim != 2:
                raise ValueError("%s needs %s clips [L, C], got %s %r"
                                 % (call, " or ".join(str(np.dtype(d)) for d in dtypes), a.dtype, a.shape))
            ps.append(np.ascontiguousarray(a))
        if not np.isscalar(sample_rate):
            rates = list(sample_rate)
            if len(rates) != len(ps) or any(r != rates[0] for r in rates):
                raise ValueError("%s takes one sample rate per call, got %r for %d clips" % (call, rates, len(ps)))
            sample_rate = rates[0] if rates else MODEL_RATE
        if sample_rate != MODEL_RATE:
            check_resample_rates(sample_rate, MODEL_RATE)   # the rate is refused before any library call
        if not ps:
            return ps, 0, (), sample_rate
        ch = ps[0].shape[1]
        if any(p_.shape[1] != ch for p_ in ps):
            raise ValueError("all clips of a batch must have the same channel count, got %r" % sorted({p_.shape[1] for p_ in ps}))
        if not 1 <= ch <= 16:
            raise ValueError("%s takes 1 to 16 channels, got %d" % (call, ch))
        if wiener:
            check_wiener_channels(ch)
        return ps, ch, (ch, int(wiener), int(wiener_radius)), sample_rate

    def _pcm16_batch(self, entry, ps, outs, channels, args, pre=(), dtype=np.int16):
        """clips ps through the multi-clip entry point `entry` -> outs, `dtype` [nsrc, L, *channels] each (made when
        None).  args: the entry's arguments between the clip lengths and scale_factor; pre: those between the plan and
        the clip count."""
        n = len(ps)
        Ls = np.array([p_.shape[0] for p_ in ps], dtype=np.int64)
        if outs is None:
            outs = [np.empty((self.nsrc, int(L)) + channels, dtype=dtype) for L in Ls]
        assert all(o.dtype == dtype and o.shape == (self.nsrc, int(L)) + channels and o.flags.c_contiguous
                   for o, L in zip(outs, Ls))
        pin = (C.c_void_p * n)(*[p_.ctypes.data for p_ in ps])
        pout = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        _lib.check(entry(self.ctx.handle, self.model.handle, self.stft.handle, *pre, n, pin, Ls.ctypes.data, *args,
                         self.scale_factor, self.overlap, self.patcher, pout, Ls.ctypes.data,
                         _stream_ptr(None, self.ctx.device)))
        return outs

    # ---- device buffers (torch tensors) ----
    def separate_device(self, audio, out=None, stream=None):
        """audio: torch float32 cuda [L] -> torch float32 cuda [nsrc, L]; asynchronous."""
        import torch
        L = audio.numel()
        if out is None:
            out = torch.empty((self.nsrc, L), dtype=torch.float32, device=audio.device)
        _lib.check(self.lib.dcs_separate_audio(self.ctx.handle, self.model.handle, self.stft.handle, _ptr(audio), L,
                                               self.scale_factor, self.overlap, self.patcher, _ptr(out), out.stride(0),
                                               _stream_ptr(stream, self.ctx.device)))
        return out

    def separate_score(self, audio, filters, out=None, stream=None, sample_rate=MODEL_RATE):
        """Score-informed Bach10: audio float [L] (numpy or cuda tensor) + normalised score filters
        [4, T, F] float32 (deepconvsep_b200.score.score_filters; or a cuda tensor [4, T, ldf] already on the
        device) -> stems float32 [4, L] (same kind as `audio`).  The four input channels are formed on the device.
        sample_rate other than 44.1 kHz is refused: the score is on the 44.1 kHz frame grid."""
        check_model_rate(sample_rate, "separate_score", _SCORE_AT_RATE)
        import torch
        host = not hasattr(audio, "is_cuda")
        T = self.stft.num_frames(np.size(audio) if host else audio.numel())
        if hasattr(filters, "is_cuda"):      # already on the device, padded rows: [4, T, ldf] float32
            fd = filters
            assert fd.is_cuda and fd.dtype == torch.float32 and fd.is_contiguous() and tuple(fd.shape) == (4, T, self.stft.ldf)
        else:
            dev = self.stft.dev if host else audio.device
            f = np.asarray(filters, dtype=np.float32)
            assert f.shape == (4, T, self.model.F), (f.shape, (4, T, self.model.F))
            fd = torch.zeros((4, T, self.stft.ldf), dtype=torch.float32, device=dev)
            fd[:, :, :self.model.F] = torch.as_tensor(f, device=dev)
        return self._score_clip(self.lib.dcs_separate_audio_score, audio, (_ptr(fd),), out, stream)

    def separate_notes(self, audio, melody, frame0=0, out=None, stream=None, sample_rate=MODEL_RATE):
        """separate_score with the filters rasterised on the device from the note table (dcs_separate_audio_notes):
        audio float [L] (numpy or cuda tensor) + melody float64 [4, nnotes, ncols] (deepconvsep_b200.score.score_melody)
        -> stems float32 [4, L] (same kind as `audio`), the bits of separate_score(audio, filterSpec(..., frame0,
        frame0 + T)).  frame0: the table frame of the clip's first STFT frame (a segment of a longer recording).
        sample_rate other than 44.1 kHz is refused: the note table is on the 44.1 kHz frame grid."""
        check_model_rate(sample_rate, "separate_notes", _SCORE_AT_RATE)
        if self.model.arch not in ("bach10_score", "bach10_score_1x1"):
            raise ValueError("separate_notes needs a score-informed network, this one is %r" % self.model.arch)
        if int(frame0) < 0:
            raise ValueError("frame0 %d must be >= 0" % frame0)
        m = check_melody(melody, 4)
        return self._score_clip(self.lib.dcs_separate_audio_notes, audio, (m.ctypes.data, m.shape[1], m.shape[2], int(frame0)),
                                out, stream)

    def _score_clip(self, entry, audio, args, out, stream):
        """audio float [L] (numpy, or a cuda tensor) through the score-informed clip entry point `entry` -> stems
        float32 [nsrc, L], numpy for numpy audio.  args: the entry's arguments between the clip length and
        scale_factor."""
        import torch
        host = not hasattr(audio, "is_cuda")
        x = torch.as_tensor(np.ascontiguousarray(audio, dtype=np.float32), device=self.stft.dev) if host else audio
        L = x.numel()
        outd = out if (out is not None and not host) else torch.empty((self.nsrc, L), dtype=torch.float32, device=x.device)
        _lib.check(entry(self.ctx.handle, self.model.handle, self.stft.handle, _ptr(x), L, *args, self.scale_factor,
                         self.overlap, self.patcher, _ptr(outd), outd.stride(0), _stream_ptr(stream, self.ctx.device)))
        return outd.cpu().numpy() if host else outd

    def separate_stereo(self, audio, out=None, stream=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE):
        """Stereo / ILD network (examples/dsd100_2ch_ILD/trainCNN_ILD_DSD100.py:299-327): audio float
        [L, 2] (numpy) or [2, L] (cuda tensor) -> `sep_audio` float32 [L, nsrc, 2] (numpy) or the device
        planes [nsrc * 2, L] ordered (source, channel) (cuda tensor in -> cuda tensor out).  wiener: EM iterations of
        the multichannel Wiener post-filter (dcs_set_wiener) on the network's spectra, 0 = off; wiener_radius: its
        covariance window in chunks to either side (dcs_set_wiener_radius), 0 = the whole clip.  sample_rate: as in
        separate (resampled to 44.1 kHz and back on the device at other rates)."""
        return self._two_channel_clip(self.lib.dcs_separate_audio_stereo, audio, out, stream, wiener, wiener_radius,
                                      sample_rate, self.separate_stereo)

    def separate_keep_channels(self, audio, out=None, stream=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE):
        """Stereo stems from the DSD100 / hiphopss network (dcs_separate_audio_keep_channels): the network sees the
        downmix (l + r) * 0.5, its soft masks are applied to each channel's STFT and inverted with that channel's
        phase.  audio float [L, 2] (numpy) or [2, L] (cuda tensor) -> float32 [L, nsrc, 2] (numpy, the layout of
        separate_stereo) or the device planes [nsrc * 2, L] ordered (source, channel) (cuda tensor in -> out).
        wiener: EM iterations of the multichannel Wiener post-filter (dcs_set_wiener) on the masked spectra, 0 = off;
        wiener_radius: its covariance window in chunks to either side (dcs_set_wiener_radius), 0 = the whole clip.
        sample_rate: as in separate (resampled to 44.1 kHz and back on the device at other rates)."""
        return self._two_channel_clip(self.lib.dcs_separate_audio_keep_channels, audio, out, stream, wiener, wiener_radius,
                                      sample_rate, self.separate_keep_channels)

    def _two_channel_clip(self, entry, audio, out, stream, wiener, wiener_radius, sample_rate=MODEL_RATE, method=None):
        """audio float [L, 2] (numpy) or [2, L] (cuda tensor) through the two-channel clip entry point `entry`, with
        `wiener` EM iterations of the Wiener post-filter over covariance windows of `wiener_radius` chunks -> float32
        [L, nsrc, 2] (numpy) or the device planes [nsrc * 2, L] ordered (source, channel) (cuda tensor in -> out).
        At another sample_rate: `method`, the public call of `entry`, on the audio resampled to MODEL_RATE."""
        check_wiener_radius(wiener, wiener_radius)
        if sample_rate != MODEL_RATE:
            return self._at_rate(partial(method, wiener=wiener, wiener_radius=wiener_radius), audio, sample_rate, out,
                                 stream, channels=2)
        host, x, outd = self._channel_planes(audio, out, self.nsrc, 2)
        L = x.shape[1]
        self.ctx.set_wiener(wiener)
        self.ctx.set_wiener_radius(wiener_radius)
        _lib.check(entry(self.ctx.handle, self.model.handle, self.stft.handle, _ptr(x), x.stride(0), L, self.scale_factor,
                         self.overlap, self.patcher, _ptr(outd), outd.stride(0), _stream_ptr(stream, self.ctx.device)))
        return self._channel_stems(host, outd, out, 2)

    def _channel_planes(self, audio, out, nsrc, channels=None):
        """The marshalling of every multi-channel clip call: audio float [L, C] (numpy) or [C, L] (cuda tensor), C =
        `channels` when given, else 1..16 -> (host: audio was numpy, x: float32 cuda planes [C, L], outd: the device stem
        planes [nsrc * C, L], `out` itself for cuda audio)."""
        import torch
        host = not hasattr(audio, "is_cuda")
        want = "%d" % channels if channels else "1 to 16"
        if host:
            a = np.asarray(audio, dtype=np.float32)
            if a.ndim != 2 or not (a.shape[1] == channels if channels else 1 <= a.shape[1] <= 16):
                raise ValueError("this call needs audio [L, C] with C = %s channels%s, got shape %r"
                                 % (want, " (two-channel separation needs stereo audio [L, 2])" if channels == 2 else "", a.shape))
            x = torch.as_tensor(np.ascontiguousarray(a.T), device=self.stft.dev)
        else:
            x = audio.contiguous()
            if x.dim() != 2 or x.dtype != torch.float32 or not (x.shape[0] == channels if channels else 1 <= x.shape[0] <= 16):
                raise ValueError("this call needs float32 device planes [C, L] with C = %s channels, got %r %s"
                                 % (want, tuple(x.shape), x.dtype))
        if x.shape[0] == 1:
            x = x.reshape(-1).unsqueeze(0)       # a single plane still reports a plane stride of L
        C_, L = x.shape
        if out is not None and not host:
            assert out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (nsrc * C_, L) and out.stride(1) == 1
            return host, x, out
        return host, x, torch.empty((nsrc * C_, L), dtype=torch.float32, device=x.device)

    @staticmethod
    def _channel_stems(host, outd, out, channels):
        """device stem planes [nsrc * C, L] ordered (source, channel) -> as they are (cuda audio), or float32
        [L, nsrc, C] numpy (into `out` when given)"""
        if not host:
            return outd
        nplanes, L = outd.shape
        stems = outd.cpu().numpy().reshape(nplanes // channels, channels, L).transpose(2, 0, 1)
        if out is not None:
            out[...] = stems
            return out
        return np.ascontiguousarray(stems)

    def separate_channels(self, audio, out=None, stream=None, wiener=0, wiener_radius=0, sample_rate=MODEL_RATE):
        """Stems for any number of channels from a single-channel network (dcs_separate_audio_channels): the network
        sees the downmix (((a_0 + a_1) + a_2) + ...) * (1 / C) in fp32, its blended soft masks are applied to the STFT
        of every channel inside the inverse STFT -- no masked spectra in memory, a workspace that does not grow with C.
        audio float [L, C] (numpy) or [C, L] (cuda tensor), C in 1..16 -> float32 [L, nsrc, C] (numpy; at C = 2 the
        layout and, for the DSD100 network, the bits of separate_keep_channels) or the device planes [nsrc * C, L]
        ordered (source, channel).  No spectrum tap; the stereo / ILD and score-informed networks are refused:
        separate_masks + apply_masks serve them.
        wiener > 0 (C in 2..8): that many EM iterations of the multichannel Wiener post-filter on the masked spectra
        M_s * X_c, over covariance windows of wiener_radius chunks to either side (0 = the whole clip), between the
        masks and the inverse STFT (dcs_separate_audio_channels_wiener); the spectra are then in memory, so the
        workspace grows with C.  At C = 2 with the DSD100 network, the bits of separate_keep_channels with the same
        wiener and wiener_radius.
        sample_rate: as in separate (resampled to 44.1 kHz and back on the device at other rates, all C channels and
        then all nsrc * C stem planes in one launch each)."""
        check_channels_family(self.model.arch)
        check_wiener_radius(wiener, wiener_radius)
        if wiener < 0:
            raise ValueError("wiener %d: the number of EM iterations cannot be negative" % wiener)
        if wiener:
            shape = np.shape(audio) if not hasattr(audio, "is_cuda") else tuple(audio.shape)[::-1]
            check_wiener_channels(shape[1] if len(shape) == 2 else 1)
        if sample_rate != MODEL_RATE:
            return self._at_rate(partial(self.separate_channels, wiener=wiener, wiener_radius=wiener_radius), audio,
                                 sample_rate, out, stream)
        host, x, outd = self._channel_planes(audio, out, self.nsrc)
        C_, L = x.shape
        if wiener:
            _lib.check(self.lib.dcs_separate_audio_channels_wiener(
                self.ctx.handle, self.model.handle, self.stft.handle, _ptr(x), C_, x.stride(0), L, self.scale_factor,
                self.overlap, self.patcher, int(wiener), int(wiener_radius), _ptr(outd), outd.stride(0),
                _stream_ptr(stream, self.ctx.device)))
        else:
            _lib.check(self.lib.dcs_separate_audio_channels(self.ctx.handle, self.model.handle, self.stft.handle, _ptr(x), C_,
                                                            x.stride(0), L, self.scale_factor, self.overlap, self.patcher,
                                                            _ptr(outd), outd.stride(0), _stream_ptr(stream, self.ctx.device)))
        return self._channel_stems(host, outd, out, C_)

    def apply_masks(self, audio, masks, out=None, stream=None, sample_rate=MODEL_RATE):
        """The caller's masks -- separate_masks' of any network, edited or not -- applied to every channel of `audio`
        inside the inverse STFT (dcs_apply_masks): plane (s, c) = iSTFT(masks_s * STFT(channel c)).  audio float [L, C]
        (numpy) with masks [nsrc, T, F], or device planes [C, L] with masks float32 cuda [nsrc, T, ldf] (planes may be
        views with gaps, rows contiguous; pad columns are not read) -> float32 [L, nsrc, C] (numpy) or the device
        planes [nsrc * C, L] ordered (source, channel).  nsrc is the masks' own: any number >= 1.
        sample_rate other than 44.1 kHz is refused: the masks are on the 44.1 kHz STFT grid."""
        check_model_rate(sample_rate, "apply_masks", _MASKS_AT_RATE)
        import torch
        host = not hasattr(audio, "is_cuda")
        L = np.shape(audio)[0] if host else audio.shape[-1]
        T, ldf, F = self.stft.num_frames(L), self.stft.ldf, self.stft.F
        if host:
            m = np.asarray(masks, dtype=np.float32)
            if m.ndim != 3 or m.shape[0] < 1 or tuple(m.shape[1:]) != (T, F):
                raise ValueError("apply_masks needs masks [nsrc, T, F] = [nsrc, %d, %d] for this audio, got %r" % (T, F, m.shape))
            md = torch.zeros((m.shape[0], T, ldf), dtype=torch.float32, device=self.stft.dev)
            md[:, :, :F] = torch.as_tensor(m, device=self.stft.dev)
        else:
            md = masks
            if not (md.is_cuda and md.dtype == torch.float32 and md.dim() == 3 and md.shape[0] >= 1 and
                    tuple(md.shape[1:]) == (T, ldf) and md.stride(2) == 1 and md.stride(1) == ldf):
                raise ValueError("apply_masks needs float32 device masks [nsrc, T, ldf] = [nsrc, %d, %d] with contiguous "
                                 "rows for this audio, got %r" % (T, ldf, tuple(md.shape)))
        nsrc = int(md.shape[0])
        host, x, outd = self._channel_planes(audio, out, nsrc)
        C_ = x.shape[0]
        _lib.check(self.lib.dcs_apply_masks(self.ctx.handle, self.stft.handle, _ptr(x), C_, x.stride(0), L, _ptr(md), nsrc,
                                            md.stride(0), _ptr(outd), outd.stride(0), _stream_ptr(stream, self.ctx.device)))
        return self._channel_stems(host, outd, out, C_)

    def separate_masks(self, audio, filters=None, melody=None, frame0=0, out=None, stream=None, sample_rate=MODEL_RATE):
        """The network's blended soft masks, from a pipeline that stops before the inverse STFT (dcs_separate_masks*):
        the fp32 values the stems calls multiply by the mixture STFT, so Stft.inverse(X * masks) gives the stems.
        audio as the stems call of this network takes it -- float [L] (single-channel nets), [L, 2] numpy or [2, L] cuda
        tensor (stereo / ILD net); score-informed nets also need the score filters `filters` (as separate_score) or the
        note table `melody` from table frame `frame0` (as separate_notes).  numpy in -> float32 [nsrc, T, F] ([nsrc, 2,
        T, F] for the stereo net); cuda tensor in -> the device planes [nplanes, T, ldf] (or into `out`, whose rows must be
        contiguous; its pad columns and the gaps between planes are not written), planes ordered (source, channel).
        sample_rate other than 44.1 kHz is refused: the masks are on the 44.1 kHz STFT grid."""
        check_model_rate(sample_rate, "separate_masks", _MASKS_AT_RATE)
        import torch
        arch = self.model.arch
        score = arch in ("bach10_score", "bach10_score_1x1")
        if melody is not None and not score:
            raise ValueError("separate_notes needs a score-informed network, this one is %r" % arch)
        if filters is not None and not score:
            raise ValueError("separate_score needs a score-informed network, this one is %r" % arch)
        if score and (filters is None) == (melody is None):
            raise ValueError("the score-informed network %r needs either the score filters or the note table" % arch)
        if int(frame0) < 0:
            raise ValueError("frame0 %d must be >= 0" % frame0)
        host = not hasattr(audio, "is_cuda")
        stereo = arch == "dsd_ild"
        if host:
            a = np.asarray(audio, dtype=np.float32)
            if stereo and (a.ndim != 2 or a.shape[1] != 2):
                raise ValueError("the stereo network needs stereo audio [L, 2], got shape %r" % (a.shape,))
            if not stereo and a.ndim != 1:
                raise ValueError("this network needs mono audio [L], got shape %r" % (a.shape,))
            x = torch.as_tensor(np.ascontiguousarray(a.T if stereo else a), device=self.stft.dev)
        else:
            x = audio.contiguous()
            assert x.dtype == torch.float32 and x.dim() == (2 if stereo else 1) and (not stereo or x.shape[0] == 2)
        L = x.shape[-1]
        T, ldf, nplanes = self.stft.num_frames(L), self.stft.ldf, self.nsrc * (2 if stereo else 1)
        if out is not None and not host:
            assert out.is_cuda and out.dtype == torch.float32 and out.dim() == 3 and tuple(out.shape[1:]) == (T, ldf)
            assert out.shape[0] == nplanes and out.stride(2) == 1 and out.stride(1) == ldf
            outd = out
        else:
            outd = torch.empty((nplanes, T, ldf), dtype=torch.float32, device=x.device)
        tail = (self.scale_factor, self.overlap, self.patcher, _ptr(outd), outd.stride(0), _stream_ptr(stream, self.ctx.device))
        h, m, p = self.ctx.handle, self.model.handle, self.stft.handle
        if melody is not None:
            mel = check_melody(melody, 4)
            _lib.check(self.lib.dcs_separate_masks_notes(h, m, p, _ptr(x), L, mel.ctypes.data, mel.shape[1], mel.shape[2],
                                                         int(frame0), *tail))
        elif filters is not None:
            if hasattr(filters, "is_cuda"):
                fd = filters
                assert fd.is_cuda and fd.dtype == torch.float32 and fd.is_contiguous() and tuple(fd.shape) == (4, T, ldf)
            else:
                f = np.asarray(filters, dtype=np.float32)
                assert f.shape == (4, T, self.model.F), (f.shape, (4, T, self.model.F))
                fd = torch.zeros((4, T, ldf), dtype=torch.float32, device=x.device)
                fd[:, :, :self.model.F] = torch.as_tensor(f, device=x.device)
            _lib.check(self.lib.dcs_separate_masks_score(h, m, p, _ptr(x), L, _ptr(fd), *tail))
        else:
            _lib.check(self.lib.dcs_separate_masks(h, m, p, _ptr(x), x.stride(0) if stereo else L, L, *tail))
        if not host:
            return outd
        M = outd[:, :, :self.model.F].cpu().numpy()
        M = M.reshape(self.nsrc, 2, T, self.model.F) if stereo else M
        if out is not None:
            out[...] = M
            return out
        return M

    def separate_tapped(self, audio, filters=None, pool=False, keep_channels=False, wiener=0, melody=None, frame0=0,
                        wiener_radius=0):
        """Parity-test entry: the whole-clip call clip_call() picks for these inputs (separate() / separate_score() /
        separate_notes() / separate_stereo() / separate_keep_channels()) with the spectrum tap on
        (dcs_set_spectrum_tap) -> (stems as that call returns them, masked spectra complex64 numpy [nplanes, T, F] --
        the tensors the inverse STFT of THIS call consumed, (source, channel) planes for the stereo outputs).
        pool=True: also the routing decisions of this call (dcs_set_pool_tap) -- max-pool net: the tie bits uint8
        [T, WP, 32]; 1x1 score net: the gate codes of conv1..conv6, a list of uint8 [rows, W, C] (gate_code_layout).
        wiener: EM iterations of the Wiener post-filter (two-channel stems only), wiener_radius its covariance window;
        the tap then holds the filtered spectra.  keep_channels without the filter forms no masked spectra in the
        library: S is built here from the masks of the (l + r) * 0.5 downmix times each channel's STFT, componentwise in
        fp32 -- the products the masked inverse STFT consumed.
        melody (score-informed nets): the note table instead of `filters`, through separate_notes(audio, melody, frame0)."""
        import torch
        run = clip_call(self, filters, melody, frame0, keep_channels, wiener, wiener_radius)
        a = np.asarray(audio)
        L = a.shape[0]
        T = self.stft.num_frames(L)
        if keep_channels and not wiener:
            out = run(a)
            x = torch.as_tensor(np.ascontiguousarray(a.T, dtype=np.float32), device=self.stft.dev)
            M = self.separate_masks((x[0] + x[1]) * 0.5)
            X = [torch.view_as_real(self.stft.forward(x[c], want_mag=False)[0]) for c in range(2)]
            S = torch.view_as_complex(torch.stack([X[c] * M[s, :, :, None] for s in range(self.nsrc) for c in range(2)]))
            return out, S[:, :, :self.model.F].cpu().numpy()
        nplanes = self.nsrc * (2 if self.model.arch == "dsd_ild" or keep_channels else 1)
        tap = torch.zeros((nplanes, T, self.stft.ldf), dtype=torch.complex64, device=self.stft.dev)
        _lib.check(self.lib.dcs_set_spectrum_tap(self.ctx.handle, _ptr(tap), tap.numel()))
        bits = None
        if pool:
            assert self.model.arch in ("ikala", "bach10_score_1x1"), "only the max-pool and 1x1 score nets have routing decisions to tap"
            if self.model.arch == "ikala":
                WP = ((self.model.F - 30) // 3 + 1) // 4
                bits = torch.zeros((T, WP, 32), dtype=torch.uint8, device=self.stft.dev)
            else:
                layout = gate_code_layout(self.model.F, self.model.tc, self._frames_spanned(T))
                bits = torch.zeros(sum(r * w * c for r, w, c in layout), dtype=torch.uint8, device=self.stft.dev)
            _lib.check(self.lib.dcs_set_pool_tap(self.ctx.handle, _ptr(bits), bits.numel()))
        try:
            out = run(a)
            torch.cuda.synchronize(self.stft.dev)
        finally:
            _lib.check(self.lib.dcs_set_spectrum_tap(self.ctx.handle, None, 0))
            _lib.check(self.lib.dcs_set_pool_tap(self.ctx.handle, None, 0))
        S = tap[:, :, :self.model.F].cpu().numpy()
        if pool and self.model.arch == "bach10_score_1x1":
            flat, codes = bits.cpu().numpy(), []
            for r, w, c in gate_code_layout(self.model.F, self.model.tc, self._frames_spanned(T)):
                codes.append(flat[:r * w * c].reshape(r, w, c))
                flat = flat[r * w * c:]
            return out, S, codes
        return (out, S, bits.cpu().numpy()) if pool else (out, S)

    def _frames_spanned(self, T):
        """Tp: the frames the patches of a T-frame clip span (dcs.h, dcs_set_pool_tap)"""
        P, step = self.num_patches(T), self.model.tc - self.overlap
        return max(T, (P - 1) * step + self.model.tc)

    def separate_spec(self, mag, X, stream=None):
        """scaled magnitude [T, ldf] + mixture STFT [T, ldf] -> masked spectra complex64 [nsrc, T, ldf]"""
        import torch
        T, ldf = mag.shape
        S = torch.empty((self.nsrc, T, ldf), dtype=torch.complex64, device=mag.device)
        _lib.check(self.lib.dcs_separate_spec(self.ctx.handle, self.model.handle, _ptr(mag), _ptr(X), T, ldf, self.overlap,
                                              self.patcher, _ptr(S), T * ldf, _stream_ptr(stream, self.ctx.device)))
        return S

    def num_patches(self, T):
        return int(self.lib.dcs_num_patches(int(T), self.model.tc, self.overlap, self.patcher))
