"""fp64 restatement of the resampler's formula (include/fs2b200.h, fastspeech2_b200/resample.py), for the tests only:

    y[j] = sum_i x[i] * h[j * down - i * up + half_len],  0 <= i < n,  0 <= j * down - i * up + half_len <= 2 half_len,

for j < ceil(n * up / down), half_len = (len(h) - 1) / 2.  Evaluated per output over its K = ceil(len(h) / up) polyphase taps."""
import numpy as np


def resample_ref(x, h, up, down):
    """x: [n] or [B, n] input, h: the full filter (fp64, firwin(...) * up); returns [ceil(n up / down)] (or [B, ...]) fp64."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 2:
        return np.stack([resample_ref(r, h, up, down) for r in x])
    h = np.asarray(h, dtype=np.float64)
    n, half_len = x.shape[0], (len(h) - 1) // 2
    K = -(-len(h) // up)
    hp = np.zeros(K * up)
    hp[:len(h)] = h
    hp = hp.reshape(K, up).T                                   # hp[p, k] = h[p + k * up]
    n_out = -(-n * up // down)
    s = np.arange(n_out, dtype=np.int64) * down + half_len
    q, p = s // up, s % up
    xp = np.concatenate([np.zeros(K), x, np.zeros(K)])        # xp[i + K] = x[i], zero outside [0, n)
    y = np.zeros(n_out)
    for k in range(K):
        i = q - k
        y += hp[p, k] * xp[np.clip(i, -K, n + K - 1) + K]
    return y
