"""Drop-in for examples/bach10_scoreinformed/separate_bach10.py: score-informed separation of
bassoon / clarinet / saxophone / violin.

    python -m deepconvsep_b200.examples.bach10_scoreinformed.separate_bach10 -i <inputfile> -o <outputdir> -m <path_to_model.pkl>

The scores are read from the directory of the input file: `bassoon_b.txt`, `clarinet_b.txt`,
`saxophone_b.txt`, `violin_b.txt`, one `onset,offset,note` line per note (README.md:50,176).

The reference script is not runnable as shipped (undefined `sources`, `util`, `toverlap`, `output`,
`bisect_right`, ... -- SURVEY.md 0.8); the working definition of this path is the separation branch
of trainCNNrwc.py:357-416, which this module follows: util's zero-padded patcher, the mixture
estimate is the SUM of the four input channels, masks use channels 0..3 of the concat output."""
import os
import sys
import getopt
import numpy as np
import scipy.io.wavfile

from ...models import load_model, infer_arch           # noqa: F401
from ...transform import sinebell, stft_norm, istft_norm, transformFFT  # noqa: F401
from ...util import generate_overlapadd, overlapadd_multi  # noqa: F401  (util.py:220-327)
from ...score import str2midi, getMidiNum, expandMidi, filterSpec, slicefft_slices, score_filters, score_melody  # noqa: F401
from ...engine import Separator
from .. import _common

FAMILY = "bach10_score"
USAGE = 'python separate_bach10.py -i <inputfile> -o <outputdir> -m <path_to_model.pkl>'
SOURCES = ['bassoon', 'clarinet', 'saxphone', 'violin']
SOURCES_MIDI = ['bassoon_b', 'clarinet_b', 'saxophone_b', 'violin_b']
_cache = {}


def build_ca(input_var=None, batch_size=32, time_context=30, feat_size=513, nchannels=4):
    """trainCNNrwc.py:134-193 (4 input channels; 16 concat channels, 0..3 used)."""
    return {"arch": FAMILY, "time_context": time_context, "feat_size": feat_size, "nsources": 4, "nchannels": nchannels}


def train_auto(filein, outdir, model, scale_factor=0.3, time_context=30, overlap=20, batch_size=32, input_size=2049,
               frameSize=4096, hopSize=512):
    sampleRate, audioObj = scipy.io.wavfile.read(filein)
    if sampleRate != 44100:
        print("Sample rate is not 44100")
        return None
    audio = _common.decode(audioObj, "bach10")
    nframes = int(np.ceil(len(audio) / np.double(hopSize))) + 2
    # the note table; the filters are rasterised from it on the GPU
    melody = score_melody(os.path.dirname(os.path.abspath(filein)), SOURCES_MIDI, nframes, frameSize=frameSize,
                          hopSize=hopSize, sampleRate=sampleRate)
    key = (os.path.abspath(model), os.path.getmtime(model), scale_factor, time_context, overlap, input_size, frameSize, hopSize)
    if key not in _cache:
        _cache.clear()
        params = load_model(model)
        # build_ca (17 arrays; 11 for the one-decoder variant) or build_ca_1x1 (22 arrays): from the parameter list
        family = infer_arch(params, input_size, time_context)[0]
        _cache[key] = Separator(params, arch=family, frame_size=frameSize, hop=hopSize, window="blackmanharris",
                                scale_factor=scale_factor, time_context=time_context, overlap=overlap, patcher="util",
                                feat_size=input_size)
    stems = _cache[key].separate_notes(audio, melody)
    maxn = np.iinfo(np.int16).max
    _, filename = os.path.split(filein)
    paths = []
    for i, src in enumerate(SOURCES):
        path = os.path.join(outdir, filename.replace(".wav", "_" + src + ".wav"))
        scipy.io.wavfile.write(filename=path, rate=sampleRate, data=(stems[i].astype(np.float64) * maxn).astype('int16'))
        paths.append(path)
    return paths


def main(argv):
    try:
        opts, args = getopt.getopt(argv, "hi:o:m:", ["ifile=", "odir=", "mfile="])
    except getopt.GetoptError:
        print(USAGE)
        sys.exit(2)
    inputfile = outdir = model = None
    for opt, arg in opts:
        if opt == '-h':
            print(USAGE)
            sys.exit()
        elif opt in ("-i", "--ifile"):
            inputfile = arg
        elif opt in ("-o", "--odir"):
            outdir = arg
        elif opt in ("-m", "--mfile"):
            model = arg
    if inputfile is None or outdir is None or model is None:
        print(USAGE)
        sys.exit(2)
    train_auto(inputfile, outdir, model, 0.3, 30, 25, 32, 2049, 4096, 512)


if __name__ == "__main__":
    main(sys.argv[1:])
