"""Host-side score prelude of the score-informed Bach10 path (kept on the host, as in the reference):
note list (`onset,offset,note` text, README.md:50,176) -> per-instrument note intervals with their
harmonic-bin ranges -> normalised binary masks -> the four network input channels.

  str2midi, midi2freq, getfreqs, remove_overlap, slicefft_slices   util.py:124-191,581-605
  getMidiNum                                                       util.py:526-579
  expandMidi                                                       util.py:424-515
  filterSpec                                                       dataset.py:839-862 (LargeDatasetMask2, no timbre model)
  score_channels                                                   examples/bach10_scoreinformed/trainCNNrwc.py:364-396

The reference is Python 2: `samplerate / hop` with two ints is an INTEGER division there; it is
written `//` here.  Pinned to the reference's own functions by tests/golden/score_golden.npz."""
import os
from bisect import bisect_left, bisect_right
import numpy as np

MIDI_A4 = 69


def midi2freq(midi_number, tuning_freq=440., MIDI_A4=69.):
    return float(tuning_freq) * 2.0 ** ((float(midi_number) - float(MIDI_A4)) * (1. / 12.))


def str2midi(note_string):
    """'Bb4' -> MIDI number (util.py:581-605)"""
    if isinstance(note_string, bytes):
        note_string = note_string.decode("ascii")
    if note_string == "?":
        return float("nan")
    data = note_string.strip().lower()
    name2delta = {"c": -9, "d": -7, "e": -5, "f": -4, "g": -2, "a": 0, "b": 2}
    accident2delta = {"b": -1, "#": 1, "x": 2}
    rest = data[1:] if data[1] in accident2delta else data[2:]
    accidents = []
    for el in rest:
        if el not in accident2delta:
            break
        accidents.append(el)
    octave = int(data[len(accidents) + 1:]) if data[1] in accident2delta else int(data[1])
    return MIDI_A4 + name2delta[data[0]] + sum(accident2delta[ac] for ac in accidents) + 12 * (octave - 4)


def getfreqs(midinote, interval=30, tuning_freq=440, nharmonics=20, ismidi=True):
    factor = 2.0 ** (interval / 1200.0)
    f0 = float(midi2freq(midinote, tuning_freq=tuning_freq)) if ismidi else midinote
    fdowns = [f * f0 / float(factor) for f in range(1, nharmonics)]
    fups = [f * f0 * float(factor) for f in range(1, nharmonics)]
    return fups, fdowns


def remove_overlap(ranges):
    result = []
    current_start = current_stop = -1
    for start, stop in sorted(ranges):
        if start > current_stop:
            result.append((start, stop))
            current_start, current_stop = start, stop
        else:
            result[-1] = (current_start, stop)
            current_stop = max(current_stop, stop)
    return result


def slicefft_slices(pitch, size, interval=30, tuning_freq=440, nharmonics=20, fmin=25, fmax=18000, iscale='lin',
                    sampleRate=44100):
    """[slice(lo, hi)] of STFT bins within +-interval cents of each harmonic (util.py:171-181)"""
    if not pitch > 0:
        return []
    binfactor = float(size) / float(sampleRate)
    fups, fdowns = getfreqs(pitch, interval=interval, tuning_freq=tuning_freq, nharmonics=nharmonics)
    ranges = tuple((1 + int(np.floor(fdowns[f] * binfactor)), 1 + int(np.ceil(fups[f] * binfactor)))
                   for f in range(len(fdowns)))
    ranges = remove_overlap(ranges)
    return [slice(r[0], r[1]) for r in ranges if r[1] <= (size / 2 + 1)]


def _read_notes(instrument, FilePath):
    midifile = os.path.join(FilePath, instrument + '.txt')
    mel = np.genfromtxt(midifile, comments='!', delimiter=',', names="a,b,c", dtype=["f", "f", "S3"])
    mel = np.atleast_1d(mel)
    return mel['a'].tolist(), mel['b'].tolist(), mel['c'].tolist()


def _select(begO, endO, notes, beginTime, finishTime, tframes=None):
    """Common front of getMidiNum / expandMidi: window the note list to [beginTime, finishTime],
    clamp, drop empty / very short notes.  Returns (begin, end, notes) or None."""
    startTime = bisect_right(endO, beginTime)
    endTime = bisect_left(begO, finishTime)
    if endO[startTime] < float(beginTime):
        startTime = startTime + 1
    if endTime >= len(begO):
        endTime = len(begO) - 1
    elif begO[endTime] > float(finishTime):
        endTime = endTime - 1
    if not startTime < endTime:
        return None
    span = finishTime - beginTime
    beg = [min(max(x - beginTime, 0.0), span) for x in begO[startTime:endTime + 1]]
    end = [min(max(x - beginTime, 0.0), span) for x in endO[startTime:endTime + 1]]
    nts = list(notes[startTime:endTime + 1])
    keep = [i for i in range(len(beg))
            if not (end[i] <= 0 or end[i] <= beg[i] or (tframes is not None and beg[i] >= tframes)
                    or (end[i] - beg[i]) < 0.01)]
    return [beg[i] for i in keep], [end[i] for i in keep], [nts[i] for i in keep]


def getMidiNum(instrument, FilePath, beginTime, finishTime):
    """number of usable notes of one instrument in the time window (util.py:526-579)"""
    begO, endO, notes = _read_notes(instrument, FilePath)
    sel = _select(begO, endO, notes, beginTime, finishTime)
    return 1 if sel is None else len(sel[2])


def expandMidi(instrument, FilePath, beginTime, finishTime, interval, tuning_freq, nharmonics, samplerate, hop, window,
               timeSpan_on, timeSpan_off, nframes, fermata=0.):
    """-> intervals [notes, 2*nharmonics+3]: first frame, last frame, MIDI note, then (lo, hi) bin
    pairs of the harmonics (util.py:424-515).  None when the window holds fewer than two notes."""
    fermata = np.maximum(timeSpan_off, fermata)
    begO, endO, notes = _read_notes(instrument, FilePath)
    tframes = float(nframes) * float(hop) / float(samplerate)
    sel = _select(begO, endO, notes, beginTime, finishTime, tframes)
    if sel is None:
        return None
    beg, end, nts = sel
    fps = samplerate // hop if isinstance(samplerate, (int, np.integer)) and isinstance(hop, (int, np.integer)) \
        else samplerate / hop
    fpsr = round(float(fps))
    maxAllowed_on = int(round(timeSpan_on * float(fps)))
    maxAllowed_off = int(round(timeSpan_off * float(fps)))
    endMelody = int((finishTime - beginTime) * fpsr)
    melodyBegin, melodyEnd = [], []
    for i in range(len(end)):
        melodyBegin.append(np.maximum(0, int(beg[i] * fpsr) - maxAllowed_on))
        intersect = [mb for mb, me in zip(beg, end)
                     if (mb > beg[i]) and (me + timeSpan_off) >= (beg[i] - timeSpan_on)
                     and (mb - timeSpan_on) <= (end[i] + timeSpan_off)]
        if len(intersect) == 0:
            notesafter = [x for x in beg if (x - timeSpan_on) > (end[i] + timeSpan_off)]
            if len(notesafter) > 0:
                newoffset = np.minimum(end[i] + fermata, np.maximum(0, min(notesafter) - timeSpan_on))
            else:
                newoffset = end[i] + fermata
            melodyEnd.append(np.minimum(nframes, np.minimum(endMelody, int(newoffset * fpsr))))
        else:
            melodyEnd.append(np.minimum(nframes, np.minimum(endMelody, int(end[i] * fpsr) + maxAllowed_off)))
    melNotes = [str2midi(n) for n in nts]
    intervals = np.zeros((len(melNotes), 2 * nharmonics + 3))
    for m in range(len(melNotes)):
        intervals[m, 0] = melodyBegin[m]
        intervals[m, 1] = melodyEnd[m]
        intervals[m, 2] = melNotes[m]
        sl = slicefft_slices(melNotes[m], size=window, interval=interval, tuning_freq=tuning_freq,
                             nharmonics=nharmonics, sampleRate=samplerate)
        lo = [s.start for s in sl]
        intervals[m, 3:2 * len(lo) + 3:2] = lo
        intervals[m, 4:2 * len(lo) + 4:2] = [s.stop for s in sl]
    return intervals


def filterSpec(mag, notes, start, stop, dtype=np.float32):
    """notes [ninst, nnotes, 2*nharm+3] -> mask [T, ninst*F]: 1 on the harmonic bins of sounding
    notes, 1e-18 elsewhere, normalised over the instruments (dataset.py:839-862)."""
    ninst = notes.shape[0]
    T, F = mag.shape
    filtered = np.ones((ninst, T, F), dtype=dtype) * 1e-18
    for j in range(ninst):
        for p in range(len(notes[j])):
            if notes[j, p, 2] > 0 and np.maximum(0, np.minimum(notes[j, p, 1], stop) - np.maximum(notes[j, p, 0], start)) > 0:
                begin = int(np.maximum(notes[j, p, 0], start)) - start
                end = int(np.minimum(notes[j, p, 1], stop)) - start
                ys, ye = notes[j, p, 3::2], notes[j, p, 4::2]
                cols = [np.arange(int(ys[f]), int(ye[f])) for f in range(min(len(ys), len(ye))) if ye[f] > 0]
                if cols:
                    filtered[j, begin:end, np.hstack(cols)] = 1.
    mask = np.zeros((T, ninst * F), dtype=dtype)
    tot = np.sum(filtered, axis=0)
    for j in range(ninst):
        mask[:, j * F:(j + 1) * F] = filtered[j] / tot
    return mask


def score_melody(score_dir, instruments, nframes, frameSize=4096, hopSize=512, sampleRate=44100, nharmonics=20,
                 interval=50, tuning_freq=440, duration=40.0):
    """The note table `melody` float64 [ninst, nnotes, 2*nharmonics+3] the filters are rasterised from
    (trainCNNrwc.py:364-382: getMidiNum -> expandMidi(..., 0.2, 0.2, nframes, 0.5)); zero rows pad the
    instruments with fewer notes.  The input of Separator.separate_notes / engine.score_filters."""
    nelem = 1
    for inst in instruments:
        nelem = max(nelem, getMidiNum(inst, score_dir, 0, duration))
    melody = np.zeros((len(instruments), int(nelem), 2 * nharmonics + 3))
    for i, inst in enumerate(instruments):
        tmp = expandMidi(inst, score_dir, 0, duration, interval, tuning_freq, nharmonics, sampleRate, hopSize, frameSize,
                         0.2, 0.2, nframes, 0.5)
        if tmp is not None:
            melody[i, :tmp.shape[0], :] = tmp
    return melody


def score_filters(score_dir, instruments, nframes, feat_size, frameSize=4096, hopSize=512, sampleRate=44100,
                  nharmonics=20, interval=50, tuning_freq=440, duration=40.0):
    """The four normalised filter planes [ninst, nframes, F] the network input is built from
    (trainCNNrwc.py:364-391: filterSpec of score_melody)."""
    melody = score_melody(score_dir, instruments, nframes, frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate,
                          nharmonics=nharmonics, interval=interval, tuning_freq=tuning_freq, duration=duration)
    mask = filterSpec(np.zeros((nframes, feat_size), dtype=np.float32), melody, 0, nframes)
    return np.ascontiguousarray(mask.reshape(nframes, len(instruments), feat_size).transpose(1, 0, 2))
