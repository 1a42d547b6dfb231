"""CPU: tests/emul_cabi.py's variance head and durations make the reference's discrete decisions on every key, NaN and +-inf included.

The emulation is what the GPU tests of fs2_variance_head / fs2_durations were first written against, so it is checked here against the
torch calls the reference makes (model/modules.py:85-100, :132-135): torch.bucketize(right=False) for the pitch / energy bucket, where
ATen's search sends NaN past the last edge, and torch.clamp(round(exp(s) - 1) * c, min=0), which keeps NaN, followed by int(), which
raises on NaN / inf (counted as wild here, as the kernels count them)."""
import math

import pytest
import torch

from tests import emul_cabi as E


def bucket_keys(bins):
    """Every edge, its fp32 neighbours on both sides, +-0, subnormals, +-inf, NaN and values beyond both ends."""
    inf = torch.tensor(math.inf)
    special = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, math.inf, -math.inf, math.nan,
                            float(bins[0]) - 1.0, float(bins[-1]) + 1.0, -3.0e38, 3.0e38])
    return torch.cat([bins, torch.nextafter(bins, inf), torch.nextafter(bins, -inf), special])


BINS = {"linear": torch.linspace(-1.0, 1.0, 255), "log": torch.exp(torch.linspace(math.log(71.0), math.log(795.0), 255)),
        "straddling_zero": torch.tensor([-2.0, -1e-40, 0.0, 1e-40, 3.0])}


def same(a, b):
    """Equal values, NaN where the other is NaN."""
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def _bucket_of(x):
    return x[..., 0].long()          # emb[i] = (i, i, i, i) on a zero x: the bucket index read back exactly


@pytest.mark.parametrize("bins", list(BINS), ids=list(BINS))
def test_emulated_bucket_is_torch_bucketize(bins):
    bins = BINS[bins]
    keys = bucket_keys(bins)
    n = keys.numel()
    emb = torch.arange(bins.numel() + 1, dtype=torch.float32)[:, None].repeat(1, 4)
    x = torch.zeros(1, n, 4)
    lens = torch.tensor([n], dtype=torch.int32)
    want = torch.bucketize(keys, bins)
    assert int(want[keys.isnan()][0]) == bins.numel()            # ATen: !(edge >= NaN) everywhere, so NaN goes past the last edge
    # target path: key = target
    _, xo = E.variance_head(torch.zeros(1, n, 1), torch.zeros(1), torch.zeros(1), lens, 1.0, keys[None], bins, emb, x)
    assert torch.equal(_bucket_of(xo)[0], want)
    # prediction path (h . w + b with w = 1, b = 0 is the key itself) under scalar controls, +-inf and NaN among them
    for c in (1.0, 0.0, -1.0, math.inf, math.nan):
        pred, xo = E.variance_head(keys[None, :, None], torch.ones(1), torch.zeros(1), lens, c, None, bins, emb, x)
        assert same(pred, keys[None] * c)
        assert torch.equal(_bucket_of(xo)[0], torch.bucketize(keys * c, bins)), c


def test_emulated_durations_follow_torch_clamp_and_count_wild():
    s = torch.tensor([[0.0, math.log(1.5), math.log(2.5), math.log(3.5), 89.0, math.inf, -math.inf, math.nan, 2.0, 14.0]])
    for c in (1.0, 0.0, -1.0, 2.5, math.inf, math.nan, torch.tensor([[1.0, 1.0, 0.5, -2.0, 0.0, 1.0, 1.0, 1.0, math.nan, 1.0]])):
        d, cum, mel_len, wild = E.durations(s, False, c)
        want = torch.clamp(torch.round(torch.exp(s) - 1) * c, min=0)
        assert same(d, want), c
        bad = ~torch.isfinite(want) | (want > 1e6)
        assert wild == int(bad.sum()), c
        reps = torch.where(bad, 0, want.nan_to_num().trunc().long())
        assert torch.equal(cum.long(), reps.cumsum(1)) and int(mel_len[0]) == int(reps.sum()), c


def test_emulated_teacher_forced_durations_truncate_and_count_wild():
    t = torch.tensor([[2.7, -2.7, 0.5, -0.0, math.nan, math.inf, -math.inf, 1e6, 1e6 + 1, 3.0]])
    d, cum, mel_len, wild = E.durations(t, True, math.nan)          # d_control is not read with targets
    assert d is None and wild == 4                                    # NaN, +-inf and 1e6 + 1 (fp32: 1000001); int() raises on -inf
    assert cum[0].tolist() == [2, 2, 2, 2, 2, 2, 2, 1000002, 1000002, 1000005] and int(mel_len[0]) == 1000005
