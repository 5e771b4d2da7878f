"""One long recording over several GPUs (SURVEY.md 8(e): "for a single very long clip, split by frame
range with halo").  The reference has no such path -- `train_auto` holds the whole clip's batches in
host memory (examples/dsd100/separate_dsd.py:289-300) -- but every stage of the path is local in time,
so a recording can be cut into sample ranges that are separated independently and stitched, and the
result is the one the whole-clip pipeline produces:

* STFT frame t reads samples [tH - N/2, tH + N/2) (transform.py:309-332);
* the network sees patches of `time_context` frames on the grid k * step, step = time_context - overlap
  (separate_dsd.py:114-135, util.py:220-248);
* the sequential cross-fade makes spectrum frame f a function of the patches that cover it, from the one
  that overwrites it (offset >= overlap) onwards (separate_dsd.py:155-168);
* the inverse STFT overlap-adds the N/H frames around a sample, and its normaliser is the sum of the
  window products of the same frames (transform.py:379-394).

A segment therefore starts on a hop boundary that is also a patch boundary of the whole clip's grid
(frame0 a multiple of step), carries a left margin long enough that the first sample it contributes has
only frames of patches free of the sub-clip's own front zero padding, and a right margin for the
mirror-image condition (plan_segments documents the two bounds).  The first segment starts at sample 0 and
the last ends at the clip's end, so the true edges are reproduced by the pipeline itself.  What a segment
computes in its margins is discarded.

Two-channel stems (the stereo / ILD network, keep-channels) stitch the same way.  The multichannel Wiener
post-filter is local in time only with a sliding-window covariance (wiener_radius W >= 1, dcs_wiener_stereo_windowed):
a chunk of 128 frames is filtered from the chunks within K * W of it (K EM iterations).  Segments then start on
chunk boundaries of the whole clip too and their margins grow by K * W chunks (plan_segments).  The whole-clip
covariance (W = 0) needs the whole clip in one segment.

The arithmetic of a kept sample is that of the whole-clip run up to the summation order inside the GEMMs
(the split of K over CTAs depends on the number of patches), i.e. to float32 rounding; tests/ check the
stitched result against the whole-clip oracle at the north-star tolerance and the planner against the
oracle exactly (float64: bit-identical stitching)."""
import math
import threading
from collections import namedtuple
import numpy as np

from ._lib import WIENER_CHUNK_FRAMES as CHUNK

Segment = namedtuple("Segment", "in_start in_stop out_start out_stop frame0")


def _ceil_div(a, b):
    return -((-a) // b)


def margins(frame_size, hop, time_context, overlap, wiener_reach=0):
    """(left, right) margins in samples that plan_segments asks for (before rounding to the grids; with wiener_reach
    the right one for the least favourable position of the cut in its chunk)."""
    step = time_context - overlap
    q = _ceil_div(frame_size // 2, hop)                    # frames touched by the sub-clip's zero padding at either end
    s_v = _ceil_div(q, step) * step                        # first patch of the sub-clip without such a frame
    if wiener_reach:
        left = (_wiener_first_frame(s_v + overlap, wiener_reach) - 1) * hop + frame_size // 2
        right = (CHUNK * (wiener_reach + 1) + q + time_context - 2) * hop + frame_size // 2
        return left, right
    left = (s_v + overlap) * hop + frame_size // 2
    right = (q + time_context - 1) * hop + frame_size // 2 + hop
    return left, right


def _wiener_first_frame(exact, reach):
    """the first frame a kept sample may read when the frames from `exact` on are the whole clip's: its chunk is
    `reach` chunks after the first chunk made only of such frames"""
    return CHUNK * (_ceil_div(exact, CHUNK) + reach)


def plan_segments(num_samples, parts, frame_size, hop, time_context, overlap, wiener_reach=0):
    """Cut [0, num_samples) into at most `parts` segments.  Each Segment holds the sample range to feed the pipeline
    (in_start:in_stop), the range of the result that is kept (out_start:out_stop, absolute sample indices) and the
    index of the whole-clip STFT frame its first frame corresponds to (a multiple of step; score filters are sliced
    from there, a note table is rasterised from there).

    Left bound.  With s0 = frame0 * hop the sub-clip's frame t' is the clip's frame frame0 + t' once
    t' >= q = ceil(N/2 / hop) (no front padding inside the frame); the first patch made of such frames starts at
    s_v = ceil_step(q); the cross-fade gives the clip's value to spectrum frames f' >= s_v + overlap; a sample n' of
    the sub-clip is summed from frames t' > (n' - N/2) / hop, so n' >= (s_v + overlap) * hop + N/2 is exact.
    Right bound.  With G = (in_stop - in_start) / hop, frames t' <= G - q are free of the back padding; the last patch
    made of such frames starts at s_l = floor_step(G - q - time_context + 1); every patch covering f' < s_l + step
    exists in both runs and is exact; sample n' is summed from frames t' <= (n' + N/2) / hop, so
    n' < (s_l + step) * hop - N/2 is exact; G >= ceil((n'_stop + N/2) / hop) + q + time_context - 1 guarantees it.

    Windowed Wiener filter (wiener_reach = K * W > 0: K EM iterations, covariance windows of W chunks of CHUNK = 128
    frames).  frame0 is a multiple of lcm(step, CHUNK), so the segment's chunks are the whole clip's.  After K
    iterations chunk c is a function of the network spectra and the STFT in chunks c - K W .. c + K W (iteration k of
    chunk c' reads the window sums of chunks c' - W .. c' + W, and each of them the chunks W further out at iteration
    k - 1; the scales s_c read the STFT of the same windows), and those windows are clipped at the clip's ends only.
    So a kept sample is exact when every chunk within K W of the chunks of the frames it reads consists of exact
    frames.  Left: the exact frames are f' >= e = s_v + overlap, the first chunk made only of them is ceil(e / CHUNK),
    sample n' reads frames from a' = floor((n' - N/2) / hop) + 1 on, so n' is exact when a' >= A = CHUNK (ceil(e /
    CHUNK) + K W), i.e. n' >= (A - 1) hop + N/2.  Right: sample n' reads frames up to b' = floor((n' + N/2) / hop),
    which lie in chunk floor(b' / CHUNK); the frames f' < s_l + step are exact and s_l + step >= G - q - time_context + 2,
    so G >= B + q + time_context - 2 with B = CHUNK (floor(b' / CHUNK) + K W + 1), for the last kept sample, makes every
    frame before B exact (the STFT's exact frames t' <= G - q reach further).  Both bounds are tight to the frame: one
    chunk less on either side puts frames that differ from the whole clip's into a window the kept samples read."""
    L, N, H = int(num_samples), int(frame_size), int(hop)
    step = time_context - overlap
    assert step > 0 and L >= 0 and parts >= 1 and wiener_reach >= 0
    q = _ceil_div(N // 2, H)
    s_v = _ceil_div(q, step) * step
    left, right = margins(N, H, time_context, overlap, wiener_reach)
    align = step * CHUNK // math.gcd(step, CHUNK) if wiener_reach else step
    # no point in cores shorter than the margins they drag along
    parts = max(1, min(int(parts), L // max(1, 2 * (left + right))))
    cuts = [_ceil_div(L * r, parts * H) * H for r in range(parts)] + [L]       # cores start on hop boundaries
    segs = []
    for r in range(parts):
        o0, o1 = cuts[r], cuts[r + 1]
        if o1 <= o0:
            continue
        if wiener_reach:
            # largest aligned frame0 with o0 - frame0*H >= (A - 1)*H + N/2
            g0 = ((o0 - N // 2) // H + 1 - _wiener_first_frame(s_v + overlap, wiener_reach)) // align * align
        else:
            # largest step-aligned frame0 with o0 - frame0*H >= (s_v + overlap)*H + N/2
            g0 = ((o0 - N // 2) // H - s_v - overlap) // step * step
        if r == 0 or g0 <= 0:      # the margin reaches the clip's start: the true edge is reproduced by the pipeline itself
            g0 = 0
        s0 = g0 * H
        if r == parts - 1:
            s1 = L
        else:
            if wiener_reach:
                b = (o1 - 1 - s0 + N // 2) // H                    # the last frame the last kept sample reads
                G = CHUNK * (b // CHUNK + wiener_reach + 1) + q + time_context - 2
            else:
                G = _ceil_div(o1 - s0 + N // 2, H) + q + time_context - 1
            s1 = s0 + G * H
            if s1 >= L:
                s1 = L
        segs.append(Segment(s0, s1, o0, o1, g0))
    return segs


def stitch(segments, pieces, num_samples, dtype=np.float32):
    """pieces[i]: array [..., in_stop - in_start] of segment i (sample axis last) -> [..., num_samples]."""
    lead = pieces[0].shape[:-1]
    out = np.zeros(lead + (int(num_samples),), dtype=dtype)
    for sg, p in zip(segments, pieces):
        assert p.shape[-1] == sg.in_stop - sg.in_start, (p.shape, sg)
        out[..., sg.out_start:sg.out_stop] = p[..., sg.out_start - sg.in_start:sg.out_stop - sg.in_start]
    return out


def _geometry(sep):
    return sep.frame_size, sep.hop, sep.model.tc, sep.overlap


def _sample_axis(sep, stems, last, keep_channels=False):
    """Two-channel stems [L, nsrc, 2] (the stereo / ILD network, keep-channels) with the sample axis moved last
    (last=True: the layout the segments are stitched in) or back to the front; the other stems are sample-last
    already."""
    if not (hasattr(sep, "model") and (keep_channels or sep.model.arch == "dsd_ild")):
        return stems
    return np.ascontiguousarray(np.moveaxis(stems, 0, -1) if last else np.moveaxis(stems, -1, 0))


def _run(sep, sub, filt, melody=None, frame0=0, stereo=None):
    """One segment through a Separator's whole-clip call (engine.clip_call), or through a callable (sub, filt) ->
    array with the sample axis last (with a note table: (sub, melody, frame0)).  The note table goes to the device
    whole: each segment rasterises its own frames.  stereo: (keep_channels, wiener, wiener_radius) for clip_call."""
    if not hasattr(sep, "model"):
        return np.asarray(sep(sub, melody, frame0) if melody is not None else sep(sub, filt))
    from .engine import clip_call
    stereo = stereo or (False, 0, 0)
    return _sample_axis(sep, clip_call(sep, filt, melody, frame0, *stereo)(sub), last=True, keep_channels=stereo[0])


def _slice_filters(filters, sg, hop):
    if filters is None:
        return None
    T = _ceil_div(sg.in_stop - sg.in_start, hop) + 2            # transform.py:309
    f = filters[:, sg.frame0:sg.frame0 + T]
    assert f.shape[1] == T, (f.shape, T, sg)
    return f


def _check_inputs(seps, filters, melody, stereo):
    """The refusals made before any segment runs -> the note table as the library takes it, or None."""
    from .engine import check_stereo_options
    for sep in seps:
        if hasattr(sep, "model") and sep.model.arch == "bach10_score_1x1":
            raise ValueError("long clips are not built for the score-informed build_ca_1x1 network (bach10_score_1x1): "
                             "its segments have never been checked against the whole clip; separate the whole clip")
        if hasattr(sep, "model"):
            check_stereo_options(sep.model.arch, *stereo)
    if filters is not None and melody is not None:
        raise ValueError("pass the score as filters= or as melody=, not both")
    if melody is not None:
        from .engine import check_melody
        return check_melody(melody)
    return None


def _plan(seps_or_sep, L, parts, geometry, stereo):
    """the segments of a clip of L samples for these stereo options; whole-clip Wiener covariances over more than one
    segment are refused here, before any segment runs"""
    N, H, tc, ov = geometry if geometry is not None else _geometry(seps_or_sep)
    keep_channels, wiener, wiener_radius = stereo
    segs = plan_segments(L, parts, N, H, tc, ov, wiener_reach=wiener * wiener_radius)
    if wiener and not wiener_radius and len(segs) > 1:
        raise ValueError("the Wiener post-filter with whole-clip covariances (wiener_radius 0) needs the whole clip in one "
                         "segment, this clip is cut into %d: set wiener_radius >= 1 (a sliding-window covariance of that "
                         "many chunks of %d frames to either side) or separate the whole clip" % (len(segs), CHUNK))
    return segs, H


def separate_long(separators, audio, parts=None, filters=None, geometry=None, melody=None, keep_channels=False, wiener=0,
                  wiener_radius=0):
    """audio float [L] (stereo / ILD network and keep_channels: [L, 2]) -> what the Separator's own call returns for
    the whole clip (float32 [nsrc, L]; two-channel stems: [L, nsrc, 2]).  `separators`: one Separator or a list (one
    per GPU, or several contexts of one GPU); segment i runs on separators[i % len], one host thread per separator (the
    C-ABI calls release the GIL).  parts defaults to len(separators).  filters: score filters [4, T, F] of the whole
    clip (score-informed network), sliced per segment on the host; or melody: its note table [4, nnotes, ncols]
    (score.score_melody), which each segment rasterises on the device from its first frame on.  keep_channels, wiener,
    wiener_radius: as in Separator.separate_keep_channels / separate_stereo; wiener > 0 over more than one segment
    needs wiener_radius >= 1.  geometry=(frame_size, hop, time_context, overlap) is needed only when the separators
    are plain callables (tests)."""
    seps = list(separators) if isinstance(separators, (list, tuple)) else [separators]
    stereo = (keep_channels, wiener, wiener_radius)
    melody = _check_inputs(seps, filters, melody, stereo)
    a = np.asarray(audio)
    L = a.shape[0]
    segs, H = _plan(seps[0], L, parts or len(seps), geometry, stereo)
    pieces = [None] * len(segs)
    errors = []

    def work(w):
        try:
            for i in range(w, len(segs), len(seps)):
                sg = segs[i]
                pieces[i] = _run(seps[w], a[sg.in_start:sg.in_stop], _slice_filters(filters, sg, H), melody, sg.frame0,
                                 stereo)
        except BaseException as e:          # surfaced in the caller's thread
            errors.append(e)

    nthreads = min(len(seps), len(segs))
    if nthreads <= 1:
        work(0)
    else:
        ts = [threading.Thread(target=work, args=(w,)) for w in range(nthreads)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
    if errors:
        raise errors[0]
    return _sample_axis(seps[0], stitch(segs, pieces, L, dtype=pieces[0].dtype), last=False, keep_channels=keep_channels)


def separate_long_distributed(separator, audio, filters=None, geometry=None, group=None, melody=None, keep_channels=False,
                              wiener=0, wiener_radius=0):
    """The same (filters= or melody=, the stereo options) over the ranks of an initialised process group (one process
    per GPU, every rank holds the clip): rank r separates segments r, r + world, ...; the kept parts are gathered to
    rank 0 (sharding.gather_stems, the path's only exchange, off the data path) which returns the stitched stems;
    other ranks return None."""
    import torch.distributed as dist
    from .sharding import gather_stems
    stereo = (keep_channels, wiener, wiener_radius)
    melody = _check_inputs([separator], filters, melody, stereo)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    a = np.asarray(audio)
    L = a.shape[0]
    segs, H = _plan(separator, L, world, geometry, stereo)
    mine = []
    for i in range(rank, len(segs), world):
        sg = segs[i]
        p = _run(separator, a[sg.in_start:sg.in_stop], _slice_filters(filters, sg, H), melody, sg.frame0, stereo)
        mine.append((i, np.ascontiguousarray(p[..., sg.out_start - sg.in_start:sg.out_stop - sg.in_start])))
    gathered = gather_stems(mine, world, rank, group=group)
    if rank != 0:
        return None
    kept = dict(kv for part in gathered for kv in part)
    first = kept[0]
    out = np.zeros(first.shape[:-1] + (L,), dtype=first.dtype)
    for i, sg in enumerate(segs):
        out[..., sg.out_start:sg.out_stop] = kept[i]
    return _sample_axis(separator, out, last=False, keep_channels=keep_channels)
