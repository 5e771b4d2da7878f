"""float64 restatement of the resampling layer (deepconvsep_b200.engine.Resampler, dcs_resample): the filter
scipy.signal.resample_poly designs by default, its output as the direct sum over the input, and the rate policy."""
from math import gcd

import numpy as np
from scipy.signal import firwin

MODEL_RATE = 44100
# the rates of the policy's table: every one is accepted in both directions
TABLE_RATES = (48000, 96000, 192000, 64000, 8000, 16000, 32000, 24000, 11025, 22050, 88200, 176400)
MAX_BANK_BYTES = 112 * 1024


def ratio(rate_in, rate_out):
    """(up, down) = rate_out / rate_in in lowest terms"""
    g = gcd(rate_in, rate_out)
    return rate_out // g, rate_in // g


def taps(up, down):
    """resample_poly's default filter: firwin(2 * half_len + 1, 1 / max, window=('kaiser', 5.0)) * up, half_len = 10 max"""
    m = max(up, down)
    return firwin(2 * 10 * m + 1, 1.0 / m, window=("kaiser", 5.0)) * up


def taps_per_phase(up, down):
    return -(-(20 * max(up, down) + 1) // up)


def bank_bytes(up, down):
    return taps_per_phase(up, down) * up * 8


def accepted(rate):
    """the policy: an integer rate in [8000, 192000] whose bank to and from 44.1 kHz is at most 112 KB"""
    if rate != int(rate) or not 8000 <= rate <= 192000:
        return False
    up, down = ratio(int(rate), MODEL_RATE)
    return max(bank_bytes(up, down), bank_bytes(down, up)) <= MAX_BANK_BYTES


def length(num_in, up, down):
    return -(-num_in * up // down)


def direct(x, up, down, h, num_out=None):
    """y[..., n] = sum_j x[..., j] h[n down + half_len - j up] over 0 <= j < L and the taps, in float64, for
    n < num_out (default ceil(L up / down)); x [..., L]."""
    x = np.asarray(x, dtype=np.float64)
    h = np.asarray(h, dtype=np.float64)
    K, L = h.size, x.shape[-1]
    half = (K - 1) // 2
    n = np.arange(length(L, up, down) if num_out is None else num_out, dtype=np.int64)
    t = n * down + half
    j0, ph = t // up, t % up
    y = np.zeros(x.shape[:-1] + (n.size,))
    for i in range(-(-K // up)):
        idx, j = ph + i * up, j0 - i
        ok = (idx < K) & (j >= 0) & (j < L)
        y += np.where(ok, h[np.minimum(idx, K - 1)] * x[..., np.clip(j, 0, L - 1)], 0.0)
    return y
