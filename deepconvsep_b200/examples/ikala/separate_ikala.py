"""Drop-in for examples/ikala/separate_ikala.py: singing voice / accompaniment separation.

    python -m deepconvsep_b200.examples.ikala.separate_ikala -i <inputfile> -o <outputdir> -m <path_to_model.pkl>
"""
import sys
import numpy as np

from ...models import load_model                       # noqa: F401
from ...transform import sinebell, stft_norm, istft_norm, transformFFT  # noqa: F401
from ...util import overlapadd                         # noqa: F401  (separate_ikala.py:138-169)
from ...util import generate_overlapadd_standalone as generate_overlapadd  # noqa: F401
from .. import _common

FAMILY = "ikala"
USAGE = 'python separate_ikala.py -i <inputfile> -o <outputdir> -m <path_to_model.pkl>'


def compute_file(audio, phase=False, frameSize=1024, hopSize=512, sampleRate=44100, window=np.hanning):
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_file(
        audio, phase=phase)


def compute_inverse(mag, phase, frameSize=1024, hopSize=512, sampleRate=44100, window=np.hanning):
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_inverse(
        mag, phase)


def build_ca(input_var=None, batch_size=32, time_context=30, feat_size=1025):
    """separate_ikala.py:172-192 (conv1 30x(1,30)/3, max-pool (1,4), conv2 30x(10,20), dense 256)."""
    return {"arch": FAMILY, "time_context": time_context, "feat_size": feat_size, "nsources": 2}


def train_auto(filein, outdir, model, scale_factor=0.3, time_context=30, overlap=20, batch_size=32, input_size=513):
    """separate_ikala.py:194-256: writes <name>-voice.wav and <name>-music.wav."""
    return _common.run(FAMILY, filein, outdir, model, scale_factor, time_context, overlap, batch_size, input_size,
                       frame_size=2 * (input_size - 1), hop=512,
                       out_name=lambda fn, src: fn.replace(".wav", "-" + src + ".wav"))


def main(argv):
    """`-i -o -m` as the reference script; extra long options: see _common.parse_cli."""
    return _common.cli_main(
        argv, USAGE,
        lambda i, o, m: train_auto(i, o, m, 0.3, 30, 20, 32, 513),   # separate_ikala.py:275
        lambda f, o, m, N, w, dev, slot, several, **kw: _common.run(FAMILY, f, o, m, 0.3, 30, 20, 32, (N or 1024) // 2 + 1, frame_size=N or 1024, hop=512,
                                                     out_name=lambda fn, src: fn.replace(".wav", "-" + src + ".wav"), window=w, device=dev, slot=slot, **kw),
        family=FAMILY)


if __name__ == "__main__":
    main(sys.argv[1:])
