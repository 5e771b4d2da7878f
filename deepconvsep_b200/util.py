"""Drop-in for the hot subset of the reference's `util.py`: wav IO (util.py:40-58) and the
patch generator / cross-fade pair used by the trainers' separation branch (util.py:220-327).

In the fused CUDA pipeline (`engine.Separator`, libdcs `dcs_separate_*`) these steps never
materialise: patches are strided *views* of the per-frame encoder activations and the
cross-fade runs inside the mask kernel.  The functions below exist for callers that use them
on their own, with the reference's shapes and semantics, as vectorised numpy (host glue)."""
import numpy as np
import scipy.io.wavfile


def infoAudioScipy(filein):
    sampleRate, audioObj = scipy.io.wavfile.read(filein)
    return len(audioObj), sampleRate, audioObj.dtype


def readAudioScipy(filein):
    """-> (float audio scaled by the dtype's max, sampleRate, dtype)   (util.py:47-54)"""
    sampleRate, audioObj = scipy.io.wavfile.read(filein)
    bitrate = audioObj.dtype
    maxv = np.finfo(bitrate).max if np.issubdtype(bitrate, np.floating) else np.iinfo(bitrate).max
    return audioObj.astype('float') / maxv, sampleRate, bitrate


def writeAudioScipy(fileout, audio_out, sampleRate, bitrate="int16"):
    """(audio * iinfo(bitrate).max).astype(bitrate), no clipping   (util.py:56-58)"""
    maxn = np.iinfo(bitrate).max
    scipy.io.wavfile.write(filename=fileout, rate=sampleRate, data=(audio_out * maxn).astype(bitrate))


# ---- WAV data chunks as they are, for the C-channel batch (Separator.separate_channels_batch) ----
# readAudioScipy expands 24-bit samples to int32 on the host and cannot map them; wav_samples maps the data chunk
# itself, so a 24-bit file reaches the GPU as its own packed bytes (engine.PCM24) and is expanded there.
_WAVE_FORMAT_PCM, _WAVE_FORMAT_IEEE_FLOAT, _WAVE_FORMAT_EXTENSIBLE = 0x0001, 0x0003, 0xFFFE
# the KSDATAFORMAT_SUBTYPE_* GUIDs are the format code followed by these 14 bytes
_GUID_TAIL = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"
_U32_MAX = 0xFFFFFFFF           # also RF64's marker in place of a 32-bit size
_RIFF_LIMIT = _U32_MAX          # the largest RIFF chunk a 32-bit size holds; write_wav goes RF64 past it


def _wav_dtypes():
    from .engine import PCM24
    # (format code, bytes per sample) -> dtype of the data chunk
    return {(_WAVE_FORMAT_PCM, 2): np.dtype("<i2"), (_WAVE_FORMAT_PCM, 3): PCM24, (_WAVE_FORMAT_PCM, 4): np.dtype("<i4"),
            (_WAVE_FORMAT_IEEE_FLOAT, 4): np.dtype("<f4")}


def wav_samples(path):
    """A WAV file's samples without conversion -> (rate, samples): samples is a read-only memmap [L, C] of the data chunk,
    <i2 for 16-bit PCM, engine.PCM24 (V3, packed little-endian 3-byte samples) for a 3-byte container of at most 24
    valid bits, <i4 for 32-bit PCM, <f4 for 32-bit IEEE float.  WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT and
    WAVE_FORMAT_EXTENSIBLE (by its sub-format) headers are read, in RIFF or RF64 files (EBU Tech 3306: the sizes of the
    RIFF and data chunks in a ds64 chunk).  Any other format or sample size is refused with its code named."""
    import struct
    with open(path, "rb") as f:
        head = f.read(12)
        if len(head) < 12 or head[:4] not in (b"RIFF", b"RF64") or head[8:12] != b"WAVE":
            raise ValueError("%s: not a RIFF or RF64 WAVE file" % (path,))
        rf64 = head[:4] == b"RF64"
        ds64_data, fmt, data = None, None, None
        while fmt is None or data is None:
            ck = f.read(8)
            if len(ck) < 8:
                break
            cid, size = ck[:4], struct.unpack("<I", ck[4:])[0]
            pos = f.tell()
            if cid == b"ds64":
                ds64_data = struct.unpack("<QQQ", f.read(24))[1]   # RIFF size, data size, sample count
            elif cid == b"fmt ":
                fmt = f.read(size)
            elif cid == b"data":
                data = (pos, ds64_data if rf64 and size == _U32_MAX and ds64_data is not None else size)
            f.seek(pos + size + (size & 1))
        end = f.seek(0, 2)
    if fmt is None or data is None:
        raise ValueError("%s: no %s chunk" % (path, "fmt" if fmt is None else "data"))
    if len(fmt) < 16:
        raise ValueError("%s: fmt chunk of %d bytes" % (path, len(fmt)))
    tag, C, rate, _, align, bits = struct.unpack("<HHIIHH", fmt[:16])
    valid = bits
    if tag == _WAVE_FORMAT_EXTENSIBLE:
        if len(fmt) < 40 or fmt[26:40] != _GUID_TAIL:
            raise ValueError("%s: WAVE_FORMAT_EXTENSIBLE with an unknown sub-format GUID" % (path,))
        valid, tag = struct.unpack("<H", fmt[18:20])[0] or bits, struct.unpack("<H", fmt[24:26])[0]
    dtype = _wav_dtypes().get((tag, bits // 8)) if bits % 8 == 0 else None
    if dtype is None or valid > bits or C < 1 or align != C * dtype.itemsize:
        raise ValueError("%s: format code 0x%04x with %d-bit samples (%d valid, %d channels, block %d) is not read; "
                         "16-, 24- or 32-bit PCM (0x0001) or 32-bit float (0x0003) is" % (path, tag, bits, valid, C, align))
    offset, nbytes = data
    if offset + nbytes > end:
        raise ValueError("%s: the data chunk claims %d bytes, the file holds %d" % (path, nbytes, end - offset))
    L = nbytes // align
    if L == 0:
        return rate, np.empty((0, C), dtype=dtype)
    return rate, np.memmap(path, dtype=dtype, mode="r", offset=offset, shape=(L, C))


def write_wav(path, rate, samples, extensible=None):
    """samples [L, C] (or [L]) of the dtypes wav_samples gives (int16, engine.PCM24, int32, float32) -> a WAV file of
    them, byte for byte.  extensible: write a WAVE_FORMAT_EXTENSIBLE header (by default for more than 2 channels or
    more than 16 bits, as the format's documentation asks) or a WAVE_FORMAT_PCM / WAVE_FORMAT_IEEE_FLOAT one.  The
    file is RIFF unless it would pass 2^32 - 1 bytes; then it is RF64 (EBU Tech 3306), so 60 min of 16-channel 24-bit
    48 kHz audio (8.3 GB of samples) is written as one file."""
    import struct
    x = np.asarray(samples)
    if x.ndim == 1:
        x = x[:, None]
    le = x.dtype if x.dtype.kind == "V" else x.dtype.newbyteorder("<")
    key = {dt: k for k, dt in _wav_dtypes().items()}.get(le)
    if x.ndim != 2 or key is None or not 1 <= x.shape[1] <= 0xFFFF:
        raise ValueError("write_wav takes int16, PCM24 (V3), int32 or float32 samples [L, C], got %s %r"
                         % (x.dtype, x.shape))
    tag, b = key
    L, C = x.shape
    if extensible is None:
        extensible = C > 2 or b > 2
    if extensible:
        fmt = struct.pack("<HHIIHHHHIH", _WAVE_FORMAT_EXTENSIBLE, C, int(rate), int(rate) * C * b, C * b, 8 * b, 22, 8 * b,
                          0, tag) + _GUID_TAIL
    else:
        fmt = struct.pack("<HHIIHH", tag, C, int(rate), int(rate) * C * b, C * b, 8 * b)
    nbytes = L * C * b
    pad = nbytes & 1
    riff = 4 + 8 + len(fmt) + 8 + nbytes + pad
    rf64 = riff > _RIFF_LIMIT
    with open(path, "wb") as f:
        if rf64:
            riff += 36                 # the ds64 chunk
            f.write(b"RF64" + struct.pack("<I", _U32_MAX) + b"WAVE")
            f.write(b"ds64" + struct.pack("<IQQQI", 28, riff, nbytes, L, 0))
        else:
            f.write(b"RIFF" + struct.pack("<I", riff) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt)
        f.write(b"data" + struct.pack("<I", _U32_MAX if rf64 else nbytes))
        x = np.ascontiguousarray(x, dtype=le)
        f.write(memoryview(x.reshape(-1).view(np.uint8)))
        if pad:
            f.write(b"\x00")


def _starts(T, time_context, overlap, limit):
    step = time_context - overlap
    if step <= 0:
        raise ValueError("overlap must be smaller than time_context")
    n = 0 if T <= limit else (T - limit - 1) // step + 1
    return np.arange(n) * step


def generate_overlapadd(allmix, input_size=513, time_context=30, overlap=10, batch_size=32, sampleRate=44100):
    """[T, F] or [C, T, F] -> (fbatch [nbatches, batch_size, C, time_context, F], nchunks); a patch
    starts every time_context-overlap frames while start+overlap < T, zero padded   (util.py:220-248)"""
    allmix = np.asarray(allmix)
    assert input_size == allmix.shape[-1], "Feature size must be the same as the last dimension of the spectrogram"
    x = allmix if allmix.ndim > 2 else allmix[None]
    C, T, F = x.shape
    starts = _starts(T, time_context, overlap, overlap)
    n = len(starts)
    fbatch = np.zeros([int(np.ceil(float(n) / batch_size)), batch_size, C, time_context, F])
    if n:
        pad = np.zeros((C, starts[-1] + time_context, F))
        pad[:, :T] = x
        idx = starts[:, None] + np.arange(time_context)[None, :]
        fbatch.reshape(-1, C, time_context, F)[:n] = pad[:, idx].transpose(1, 0, 2, 3)
    return fbatch, n


def generate_overlapadd_standalone(allmix, input_size=513, time_context=30, overlap=10, batch_size=32, sampleRate=44100):
    """The stand-alone scripts' variant: while start+time_context < T, tail dropped
    (examples/dsd100/separate_dsd.py:114-135; the np.empty tail is zero here)."""
    allmix = np.asarray(allmix)
    T, F = allmix.shape
    starts = _starts(T, time_context, overlap, time_context)
    n = len(starts)
    fbatch = np.zeros([int(np.ceil(float(n) / batch_size)), batch_size, 1, time_context, F])
    if n:
        idx = starts[:, None] + np.arange(time_context)[None, :]
        fbatch.reshape(-1, 1, time_context, F)[:n, 0] = allmix[idx]
    return fbatch, n


def overlapadd_multi(fbatch, obatch, nchunks, overlap=10):
    """fbatch [nbatches, nsources, batch_size, 1, time_context, F] -> sep [nsources,
    nchunks*(time_context-overlap)+time_context, F]   (util.py:297-327)"""
    fbatch = np.asarray(fbatch)
    nsources, F, tc = fbatch.shape[1], fbatch.shape[-1], fbatch.shape[-2]
    step = tc - overlap
    patches = fbatch[:, :, :, 0].transpose(1, 0, 2, 3, 4).reshape(nsources, -1, tc, F)[:, :nchunks]
    sep = np.zeros((nsources, nchunks * step + tc, F))
    # sequential blend, vectorised over sources and bins (each step touches one patch)
    up = np.linspace(0., 1.0, num=overlap)[:, None] if overlap > 0 else np.zeros((0, 1))
    down = up[::-1]
    for k in range(nchunks):
        s = k * step
        if k == 0:
            sep[:, :tc] = patches[:, 0]
        else:
            sep[:, s + overlap:s + tc] = patches[:, k, overlap:]
            sep[:, s:s + overlap] = down * sep[:, s:s + overlap] + up * patches[:, k, :overlap]
    return sep


def overlapadd(fbatch, obatch, nchunks, overlap=10):
    """two-source variant -> (sep1, sep2)   (util.py:251-294)"""
    sep = overlapadd_multi(np.asarray(fbatch)[:, :2], obatch, nchunks, overlap=overlap)
    return sep[0], sep[1]
