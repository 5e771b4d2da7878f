"""Drop-in for examples/bach10/separate_bach10.py: bassoon / clarinet / saxophone / violin.

    python -m deepconvsep_b200.examples.bach10.separate_bach10 -i <inputfile> -o <outputdir> -m <path_to_model.pkl>
"""
import sys
from scipy.signal.windows import blackmanharris  # the reference imports scipy.signal.blackmanharris (:4)

from ...models import load_model                       # noqa: F401
from ...transform import sinebell, stft_norm, istft_norm, transformFFT  # noqa: F401
from ...util import overlapadd_multi                   # noqa: F401
from ...util import generate_overlapadd_standalone as generate_overlapadd  # noqa: F401
from .. import _common

FAMILY = "bach10"
USAGE = 'python separate_bach10.py -i <inputfile> -o <outputdir> -m <path_to_model.pkl>'


def compute_file(audio, phase=False, frameSize=1024, hopSize=512, sampleRate=44100, window=blackmanharris):
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_file(
        audio, phase=phase)


def compute_inverse(mag, phase, frameSize=1024, hopSize=512, sampleRate=44100, window=blackmanharris):
    return transformFFT(frameSize=frameSize, hopSize=hopSize, sampleRate=sampleRate, window=window).compute_inverse(
        mag, phase)


def build_ca(input_var=None, batch_size=32, time_context=30, feat_size=513):
    """separate_bach10.py:172-229 (conv1 30x(1,30)/4, conv2 30x(2T/3,1), dense 256, 4 decoders)."""
    return {"arch": FAMILY, "time_context": time_context, "feat_size": feat_size, "nsources": 4}


def train_auto(filein, outdir, model, scale_factor=0.3, time_context=30, overlap=20, batch_size=32, input_size=2049,
               frameSize=4096, hopSize=512):
    """separate_bach10.py:232-306: writes <name>_{bassoon,clarinet,saxphone,violin}.wav."""
    return _common.run(FAMILY, filein, outdir, model, scale_factor, time_context, overlap, batch_size, input_size,
                       frame_size=frameSize, hop=hopSize,
                       out_name=lambda fn, src: fn.replace(".wav", "_" + src + ".wav"))


def main(argv):
    """`-i -o -m` as the reference script; extra long options: see _common.parse_cli."""
    return _common.cli_main(
        argv, USAGE,
        lambda i, o, m: train_auto(i, o, m, 0.3, 30, 25, 32, 2049, 4096, 512),   # separate_bach10.py:325
        lambda f, o, m, N, w, dev, slot, several, **kw: _common.run(FAMILY, f, o, m, 0.3, 30, 25, 32, (N or 4096) // 2 + 1, frame_size=N or 4096, hop=512,
                                                     out_name=lambda fn, src: fn.replace(".wav", "_" + src + ".wav"), window=w, device=dev, slot=slot, **kw),
        family=FAMILY)


if __name__ == "__main__":
    main(sys.argv[1:])
