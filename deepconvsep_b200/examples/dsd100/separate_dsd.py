"""Drop-in for examples/dsd100/separate_dsd.py: DSD100 four-stem separation.

    python -m deepconvsep_b200.examples.dsd100.separate_dsd -i <inputfile> -o <outputdir> -m <path_to_model.pkl>

Same functions and signatures as the reference script; the work happens in the CUDA pipeline
(STFT -> encoder/decoder -> soft mask + cross-fade -> iSTFT), the host only reads and writes wavs."""
import sys
import numpy as np

from ...models import load_model                       # noqa: F401  (separate_dsd.py:17-21)
from ...transform import sinebell, stft_norm, istft_norm, transformFFT  # noqa: F401
from ...util import overlapadd_multi                   # noqa: F401  (separate_dsd.py:139-169)
from ...util import generate_overlapadd_standalone as generate_overlapadd  # noqa: F401  (separate_dsd.py:114-135)
from .. import _common

FAMILY = "dsd"
USAGE = 'python separate_dsd.py -i <inputfile> -o <outputdir> -m <path_to_model.pkl>'


def compute_file(audio, phase=False, frameSize=1024, hopSize=512, sampleRate=44100, window=np.hanning):
    """separate_dsd.py:24-33"""
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_file(
        audio, phase=phase)


def compute_inverse(mag, phase, frameSize=1024, hopSize=512, sampleRate=44100, window=np.hanning):
    """separate_dsd.py:36-41"""
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_inverse(
        mag, phase)


def build_ca(input_var=None, batch_size=32, time_context=30, feat_size=513):
    """separate_dsd.py:172-236 built a Lasagne graph; here the network is a fixed CUDA pipeline, so
    this returns the architecture descriptor that dcs_model_create consumes."""
    return {"arch": FAMILY, "time_context": time_context, "feat_size": feat_size, "nsources": 4,
            "layers": ["conv1 50x(1,F)", "conv2 50x(T/2,1)", "dense 128", "3 x dense 800 + InverseLayers", "bias+ReLU"]}


def train_auto(filein, outdir, model, scale_factor=0.3, time_context=30, overlap=20, batch_size=32, input_size=513):
    """separate_dsd.py:239-313: writes vocals.wav, bass.wav, drums.wav, other.wav into outdir."""
    return _common.run(FAMILY, filein, outdir, model, scale_factor, time_context, overlap, batch_size, input_size,
                       frame_size=2 * (input_size - 1), hop=512, out_name=lambda fn, src: src + ".wav")


def main(argv):
    """`-i -o -m` as separate_dsd.py:316-332; extra long options (--keep-channels, --wiener, --wiener-radius and --resample among
    them): see _common.parse_cli."""
    def run_one(f, o, m, N, w, dev, slot, several, keep_channels=False, wiener=0, wiener_radius=0, resample=False):
        # several clips into one directory: keep them apart the way the iKala / Bach10 scripts name their outputs
        name = (lambda fn, src: fn.replace(".wav", "_" + src + ".wav")) if several else (lambda fn, src: src + ".wav")
        return _common.run(FAMILY, f, o, m, 0.3, 30, 25, 32, (N or 1024) // 2 + 1, frame_size=N or 1024, hop=512,
                           out_name=name, window=w, device=dev, slot=slot, keep_channels=keep_channels, wiener=wiener,
                           wiener_radius=wiener_radius, resample=resample)
    return _common.cli_main(argv, USAGE, lambda i, o, m: train_auto(i, o, m, 0.3, 30, 25, 32, 513), run_one,
                            family=FAMILY)  # separate_dsd.py:332


if __name__ == "__main__":
    main(sys.argv[1:])
