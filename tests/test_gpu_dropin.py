"""GPU: the reference-named Python entry points (transform.transformFFT, stft_norm/istft_norm,
separate_dsd.train_auto/main) against the oracle.  fp32 device arithmetic vs float64 reference:
2e-6 relative L2 on spectra / magnitudes, 5e-6 on reconstructed audio."""
import os
import numpy as np
import pytest
import scipy.io.wavfile

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import dsp, nets, pipeline  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_transformFFT_compute_file_inverse_and_module_functions():
    from deepconvsep_b200 import transform
    rng = np.random.default_rng(0)
    x = rng.standard_normal(20000) * 0.1
    for N, H, win in [(2048, 512, np.hanning), (1024, 256, np.hanning), (4096, 512, dsp.blackmanharris)]:
        tt = transform.transformFFT(frameSize=N, hopSize=H, sampleRate=44100, window=win)
        mag, ph = tt.compute_file(x, phase=True)
        mag_r, ph_r = dsp.compute_file(x, phase=True, frameSize=N, hopSize=H, window=win)
        assert mag.dtype == np.float64 and mag.shape == mag_r.shape == ph.shape
        assert rel(mag, mag_r) < 2e-6
        assert rel(mag * np.exp(1j * ph), mag_r * np.exp(1j * ph_r)) < 3e-6
        assert rel(tt.compute_file(x), mag_r) < 2e-6
        y = tt.compute_inverse(mag_r, ph_r)
        y_r = dsp.compute_inverse(mag_r, ph_r, frameSize=N, hopSize=H, window=win)
        assert y.shape == y_r.shape and rel(y[:x.size], y_r[:x.size]) < 5e-6
        w = win(N)
        X = transform.stft_norm(x, window=w, hopsize=float(H), nfft=float(N))
        X_r = dsp.stft_norm(x, window=w, hopsize=float(H), nfft=float(N))
        assert X.dtype == np.complex128 and rel(X, X_r) < 2e-6
        y2 = transform.istft_norm(X_r, window=w, analysisWindow=w, hopsize=float(H), nfft=float(N))
        assert rel(y2[:x.size], x) < 5e-6
        # distinct synthesis / analysis windows (istft_norm's general signature)
        ws = transform.sinebell(N)
        y3 = transform.istft_norm(X_r, window=ws, analysisWindow=w, hopsize=float(H), nfft=float(N))
        y3_r = dsp.istft_norm(X_r, window=ws, analysisWindow=w, hopsize=float(H), nfft=float(N))
        assert rel(y3[:x.size], y3_r[:x.size]) < 5e-6


def test_compute_transform_dump(tmp_path):
    from deepconvsep_b200 import transform
    rng = np.random.default_rng(2)
    audio = rng.standard_normal((6000, 3)) * 0.1
    tt = transform.transformFFT(frameSize=1024, hopSize=512, suffix="f")
    mags = tt.compute_transform(audio, phase=False, save=False)
    assert mags.shape == (3, dsp.num_frames(6000, 512), 513)
    out = str(tmp_path / "song.data")
    assert tt.compute_transform(audio, out_path=out, phase=True, save=True) is None
    m = np.fromfile(str(tmp_path / "song_f_m_.data")).reshape(tt.get_shape(str(tmp_path / "song_f_m_.shape")))
    np.testing.assert_array_equal(m, mags)
    for i in range(3):
        assert rel(m[i], dsp.compute_file(audio[:, i], frameSize=1024, hopSize=512)) < 2e-6
    assert os.path.exists(str(tmp_path / "song_f_p_.data"))


def test_separate_dsd_cli_end_to_end(tmp_path):
    """python separate_dsd.py -i mix.wav -o out -m model.pkl  ==  oracle train_auto, to 1 LSB."""
    from deepconvsep_b200 import save_model
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    params = nets.make_synthetic_params("dsd", 513, seed=21)
    pkl = str(tmp_path / "model.pkl")
    save_model(pkl, params)
    mix, _ = pipeline.synth_mixture(2.5, 33)
    rng = np.random.default_rng(3)
    pcm = np.stack([np.round(mix * 30000).astype(np.int16),
                    np.round((0.8 * mix + 0.01 * rng.standard_normal(mix.size)) * 30000).astype(np.int16)], axis=1)
    wav = str(tmp_path / "mix.wav")
    scipy.io.wavfile.write(wav, 44100, pcm)
    outdir = str(tmp_path / "out")
    os.makedirs(outdir)
    separate_dsd.main(["-i", wav, "-o", outdir, "-m", pkl])
    mono = pipeline.decode_wav_array(pcm, "dsd")
    want = pipeline.separate(mono, params, "dsd", frameSize=1024, overlap=25, count_kinks=True)
    want16 = (want * 32767).astype("int16")
    for i, name in enumerate(["vocals", "bass", "drums", "other"]):
        sr, got = scipy.io.wavfile.read(os.path.join(outdir, name + ".wav"))
        assert sr == 44100 and got.dtype == np.int16 and got.shape == want16[i].shape
        d = np.abs(got.astype(np.int32) - want16[i].astype(np.int32))
        if pipeline.separate.last_kinks == 0:
            assert d.max() <= 1
        assert np.mean(d > 1) < 1e-3
    # wrong sample rate: prints and writes nothing (separate_dsd.py:313)
    scipy.io.wavfile.write(wav, 22050, pcm)
    assert separate_dsd.train_auto(wav, outdir, pkl, 0.3, 30, 25, 32, 513) is None


def test_dataset_runner_dsd100(tmp_path):
    """trainers' separation branch (dsd100/trainCNN.py:285-335): Dev/Test song folders, util patcher,
    blackmanharris analysis, stems written with the input bit depth."""
    from deepconvsep_b200 import runner
    params = nets.make_synthetic_params("dsd", 513, seed=31)
    db, out = tmp_path / "Mixtures", tmp_path / "Estimates"
    songs = {("Dev", "051 - A"): 1.7, ("Test", "001 - B"): 1.2}
    seeds = {"051 - A": 200, "001 - B": 211}     # clips for which the oracle flags no mask-discontinuity bin (fixed: hash() is salted per process)
    for (sub, name), secs in songs.items():
        mix, _ = pipeline.synth_mixture(secs, seeds[name])
        pcm = np.stack([np.round(mix * 30000), np.round(mix * 25000)], axis=1).astype(np.int16)
        os.makedirs(str(db / sub / name))
        scipy.io.wavfile.write(str(db / sub / name / "mixture.wav"), 44100, pcm)
    secs, njobs = runner.separate_dataset("dsd", str(db), str(out), params)
    assert njobs == 2 and abs(secs - 2.9) < 1e-3
    for (sub, name), _ in songs.items():
        sr, pcm = scipy.io.wavfile.read(str(db / sub / name / "mixture.wav"))
        audio = (pcm[:, 0].astype(float) / 32767 + pcm[:, 1].astype(float) / 32767) / 2
        want = pipeline.separate(audio, params, "dsd", frameSize=1024, window=dsp.blackmanharris, overlap=25,
                                 patcher="util", count_kinks=True)
        for i, s in enumerate(["vocals", "bass", "drums", "other"]):
            sr2, got = scipy.io.wavfile.read(str(out / sub / name / (s + ".wav")))
            assert sr2 == 44100 and got.dtype == np.int16
            d = np.abs(got.astype(np.int32) - (want[i] * 32767).astype("int16").astype(np.int32))
            assert pipeline.separate.last_kinks == 0
            assert d.max() <= 1                    # truncation to int16 flips at most one LSB
    # sharding: two ranks split the two songs
    assert len(runner.list_jobs("dsd", str(db), str(out))) == 2


def test_cli_long_options_directory_of_clips(tmp_path):
    """--frame-size / --window / --devices / --batch-clips (SURVEY.md 5) with -i <directory>: two clips in flight on
    device 0, every stem equal to what the plain `-i file` call writes."""
    from deepconvsep_b200 import save_model
    from deepconvsep_b200.examples.dsd100 import separate_dsd
    params = nets.make_synthetic_params("dsd", 513, seed=21)
    pkl = str(tmp_path / "model.pkl")
    save_model(pkl, params)
    indir, out1, out2 = tmp_path / "in", tmp_path / "out1", tmp_path / "out2"
    for d in (indir, out1, out2):
        os.makedirs(str(d))
    names = []
    for k, secs in enumerate((1.5, 2.2, 1.1)):
        mix, _ = pipeline.synth_mixture(secs, 40 + k)
        pcm = np.stack([np.round(mix * 30000), np.round(mix * 28000)], axis=1).astype(np.int16)
        names.append("clip%d.wav" % k)
        scipy.io.wavfile.write(str(indir / names[-1]), 44100, pcm)
    separate_dsd.main(["-i", str(indir), "-o", str(out2), "-m", pkl, "--frame-size", "1024", "--window", "hanning",
                       "--devices", "0", "--batch-clips", "2"])
    for n in names:
        separate_dsd.main(["-i", str(indir / n), "-o", str(out1), "-m", pkl])
        for src in ["vocals", "bass", "drums", "other"]:
            _, a = scipy.io.wavfile.read(str(out1 / (src + ".wav")))
            _, b = scipy.io.wavfile.read(str(out2 / n.replace(".wav", "_" + src + ".wav")))
            assert np.array_equal(a, b), (n, src)


def test_batch_scheduler_matches_per_clip_calls():
    """dcs_separate_batch_pcm16_host (H2D | kernels | D2H pipelined over the clips of a batch, double-buffered staging)
    gives the bits of dcs_separate_pcm16_host clip by clip -- different lengths, stereo input, called twice."""
    from deepconvsep_b200.engine import Separator
    params = nets.make_synthetic_params("dsd", 513, seed=12)
    sep = Separator(params, frame_size=1024, hop=512, window="hanning", overlap=25)
    rng = np.random.default_rng(1)
    clips = []
    for k, secs in enumerate((2.0, 3.1, 1.2, 2.6, 0.3)):
        mix, _ = pipeline.synth_mixture(secs, 60 + k)
        clips.append(np.stack([np.round(mix * 30000), np.round((0.7 * mix + 0.01 * rng.standard_normal(mix.size)) * 30000)],
                              axis=1).astype(np.int16))
    want = [sep.separate_pcm16(c) for c in clips]
    for _ in range(2):
        got = sep.separate_pcm16_batch(clips)
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert g.shape == w.shape and np.array_equal(g, w)
    assert sep.separate_pcm16_batch([]) == []
    # a bad clip is refused before anything is queued, and the context keeps working
    from deepconvsep_b200._lib import DcsError
    with pytest.raises(DcsError, match="clip 1"):
        sep.separate_pcm16_batch([clips[0], np.zeros((0, 2), dtype=np.int16)])
    again = sep.separate_pcm16_batch(clips[:2])
    assert np.array_equal(again[0], want[0]) and np.array_equal(again[1], want[1])


def test_refused_calls_queue_nothing():
    """A call with bad arguments is refused before it queues any work: the launch count stays where it was, and the
    context then still gives the same bits.  Covers the batch scheduler (overlap, frame size, score-informed model),
    the mono entry point with a stereo model and the score-informed entry point with overlap = time_context."""
    import ctypes as C
    from deepconvsep_b200.engine import Separator, Model, Stft
    from deepconvsep_b200._lib import DcsError, check
    params = nets.make_synthetic_params("dsd", 513, seed=12)
    sep = Separator(params, frame_size=1024, hop=512, window="hanning", overlap=25)
    lib, ctx = sep.lib, sep.ctx
    mix, _ = pipeline.synth_mixture(1.0, 61)
    clip = np.round(mix * 30000).astype(np.int16)
    want = sep.separate_pcm16(clip)
    L = clip.size
    Ls = np.array([L], dtype=np.int64)
    out16 = np.empty((4, L), dtype=np.int16)
    pin, pout = (C.c_void_p * 1)(clip.ctypes.data), (C.c_void_p * 1)(out16.ctypes.data)
    stereo = Model(ctx, nets.make_synthetic_params("dsd_ild", 513, seed=3), arch="dsd_ild", feat_size=513)
    score = Model(ctx, nets.make_synthetic_params("bach10_score", 129, seed=3), arch="bach10_score", feat_size=129)
    plan2048, plan256 = Stft(ctx, 2048, 512, "hanning"), Stft(ctx, 256, 128, "blackmanharris")
    dev = torch.device("cuda", ctx.device)
    x = torch.as_tensor(mix.astype(np.float32), device=dev)
    stems = torch.empty((8, L), dtype=torch.float32, device=dev)
    filters = torch.zeros((4, plan256.num_frames(L), plan256.ldf), dtype=torch.float32, device=dev)

    def batch(model, plan, overlap):
        return lib.dcs_separate_batch_pcm16_host(ctx.handle, model.handle, plan.handle, 1, pin, Ls.ctypes.data, 1, 0,
                                                 C.c_float(0.3), overlap, 0, pout, Ls.ctypes.data, None)

    refused = {
        "batch, overlap = time_context": lambda: batch(sep.model, sep.stft, sep.model.tc),
        "batch, plan of another frame size": lambda: batch(sep.model, plan2048, 25),
        "batch, score-informed model": lambda: batch(score, plan256, 25),
        "audio, stereo model": lambda: lib.dcs_separate_audio(ctx.handle, stereo.handle, sep.stft.handle, x.data_ptr(), L,
                                                              C.c_float(0.3), 25, 0, stems.data_ptr(), L, None),
        "score, overlap = time_context": lambda: lib.dcs_separate_audio_score(
            ctx.handle, score.handle, plan256.handle, x.data_ptr(), L, filters.data_ptr(), C.c_float(0.2), score.tc, 1,
            stems.data_ptr(), L, None),
    }
    for name, call in refused.items():
        torch.cuda.synchronize(dev)
        n0 = ctx.launch_count()
        with pytest.raises(DcsError):
            check(call())
        assert ctx.launch_count() == n0, name
    assert np.array_equal(sep.separate_pcm16(clip), want)
