"""CPU: the comparator and poison placements of tests/isolation_cases.py, the weight packing of non-finite weights, and the NaN cones of
the fp64 oracles that tests/test_gpu_isolation.py compares the kernels' NaN masks against."""
import numpy as np
import torch

from fastspeech2_b200 import configs, packing, synth
from fastspeech2_b200.hifigan import AttrDict
from fastspeech2_b200.resample import Resampler, design_taps
from oracle import fs2_oracle as O
from oracle.resample_ref import resample_ref
from tests import isolation_cases as I
from tests.generator_cases import oracle_kwargs
from tests.isolation_cases import INF, NAN, same


def test_same_compares_nan_masks_infinities_and_bits():
    a = torch.tensor([1.0, NAN, INF, -INF, 0.0, 3e38])
    assert same(a, a.clone())
    assert same(a, torch.tensor([1.0, -NAN, INF, -INF, 0.0, 3e38]))        # any NaN payload or sign is NaN
    assert not same(a, torch.tensor([1.0, 2.0, INF, -INF, 0.0, 3e38]))     # NaN mask
    assert not same(a, torch.tensor([1.0, NAN, -INF, -INF, 0.0, 3e38]))    # the sign of an infinity
    assert not same(a, torch.tensor([1.0, NAN, INF, -INF, -0.0, 3e38]))    # -0 is not +0
    assert not same(a, torch.tensor([1.0, NAN, INF, -INF, 0.0, 3e38]).nextafter(torch.tensor(0.0)))   # one ulp
    assert not same(a, a[:5]) and not same(a, a.double())
    assert same(torch.tensor([0, 255], dtype=torch.uint8), torch.tensor([0, 255], dtype=torch.uint8))
    assert not same(torch.tensor([0, 255], dtype=torch.uint8), torch.tensor([0, 213], dtype=torch.uint8))
    assert same(torch.tensor([NAN, 1.0], dtype=torch.float16), torch.tensor([NAN, 1.0], dtype=torch.float16))


def test_placements_and_cases_cover_every_poison_position_and_placement():
    assert I.rows(300, 128) == {"first": 0, "last": 299, "boundary": 128, "frame": 128, "channel": 128}
    assert I.rows(100, 128) == {"first": 0, "last": 99, "frame": 50, "channel": 50}
    assert I.rows(1, 128) == {"first": 0, "last": 0, "frame": 0, "channel": 0}
    assert I.positions(3) == [0, 1, 2] and I.positions(7) == [0, 3, 6] and I.positions(1) == [0]
    cs = I.cases(3, lambda b: 300, 128)
    assert len(cs) == 15
    assert {(p, q) for p, q, _, _ in cs} == {(p, q) for p in I.POISONS for q in range(3)}
    assert {(q, k) for _, q, k, _ in cs} == {(q, k) for q in range(3) for k in I.PLACEMENTS}
    assert all(row == I.rows(300, 128)[k] for _, _, k, row in cs)
    short = I.cases(3, lambda b: (300, 5, 300)[b], 128)
    assert all(row < (300, 5, 300)[q] for _, q, _, row in short)


def test_poison_sets_one_row_or_one_channel_of_one_tenant():
    x = torch.zeros(3, 10, 4)
    p = I.poison(x, 1, 7, NAN, "frame")
    assert torch.isnan(p[1, 7]).all() and int(torch.isnan(p).sum()) == 4 and not torch.isnan(x).any()
    p = I.poison(x, 2, 3, INF, "channel", channel=2)
    assert p[2, 3, 2] == INF and int(torch.isinf(p).sum()) == 1
    m = torch.zeros(2, 80, 6)                          # [B, C, T]
    p = I.poison(m, 0, 5, -INF, "channel", axis=2, channel=17)
    assert p[0, 17, 5] == -INF and int(torch.isinf(p).sum()) == 1
    p = I.poison(m, 1, 0, NAN, "first", axis=2)
    assert torch.isnan(p[1, :, 0]).all() and int(torch.isnan(p).sum()) == 80
    w = torch.zeros(2, 1, 9)                           # one channel: 'channel' is that channel
    assert int(torch.isnan(I.poison(w, 0, 4, NAN, "channel", axis=2, channel=5)).sum()) == 1


def test_packing_non_finite_weights_chooses_unit_scale():
    w = torch.randn(3, 32, 64, generator=torch.Generator().manual_seed(0)) * 0.01
    for v in (NAN, INF, -INF):
        wp = w.clone()
        wp[1, 5, 9] = v
        hi, lo, s = packing.split_fp16(wp)
        assert s == 1.0
        assert hi[1, 5, 9].float().isnan() if v != v else hi[1, 5, 9].float() == v
        for f8 in (False, True):
            t = packing.pack_conv_tc(wp, f8=f8)
            assert float(t[:4].view(torch.float32)[0]) == 1.0            # header: 1 / s
    assert packing.split_fp16(w)[2] != 1.0


def _intervals(mask):
    idx = mask.nonzero()[:, 0]
    return 0 if not len(idx) else 1 + int((idx[1:] - idx[:-1] > 1).sum())


def test_oracle_nan_cones_are_one_interval_per_poisoned_frame():
    """The fp64 oracle's waveform of a mel with one NaN frame (or channel) is NaN on one interval around it, about +-13 frames wide,
    and a second NaN frame far away adds a second interval."""
    h = AttrDict(configs.HIFIGAN_V2_CONFIG)
    sd = synth.hifigan_state_dict(h, seed=3)
    mel = synth.make_mel(1, 80, seed=5).double()
    for f, ch in ((40, None), (0, None), (79, 17)):
        m = mel.clone()
        if ch is None:
            m[0, :, f] = NAN
        else:
            m[0, ch, f] = NAN
        y = torch.isnan(O.hifigan_forward(sd, m, dtype=torch.float64, **oracle_kwargs("v2"))[0, 0])
        assert _intervals(y) == 1, f
        idx = y.nonzero()[:, 0]
        assert idx.min() <= 256 * f and idx.max() >= 256 * f + 255 and idx.max() - idx.min() < 256 * 30, f
    m = mel.clone()
    m[0, :, 10] = NAN
    m[0, :, 70] = NAN
    assert _intervals(torch.isnan(O.hifigan_forward(sd, m, dtype=torch.float64, **oracle_kwargs("v2"))[0, 0])) == 2


def test_resample_reference_nan_cone_is_one_interval():
    for rate in (8000, 16000, 24000, 44100):
        rs = Resampler(22050, rate)
        x = np.random.default_rng(0).standard_normal(3000) * 0.3
        for i in (0, 1500, 2999):
            xp = x.copy()
            xp[i] = np.nan
            y = np.isnan(resample_ref(xp, design_taps(rs.up, rs.down), rs.up, rs.down))
            assert _intervals(torch.from_numpy(y)) == 1, (rate, i)
            assert y.sum() <= -(-rs.K * rs.up // rs.down) + 1, (rate, i)         # the outputs whose K taps reach sample i
