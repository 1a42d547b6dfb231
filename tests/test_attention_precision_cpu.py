"""CPU: the power of tests/test_gpu_attention_precision.py, without a GPU, on the fused kernel's arithmetic emulated with exact sums
(tests/emul_cabi.py::attention_fused_emul):

  * on the plateau and pfloor rows the kernel without AF_PSCALE (P split unscaled, so its lo plane is subnormal below p ~ 2^-3) leaves the
    fused kernel's bar by at least 5x: the test catches it;
  * with AF_PSCALE every case stays within a quarter of that bar, which leaves the rest to the tensor cores' fp32 accumulation;
  * R is not vacuous: at unit magnitudes it is a fraction of the bar, and at |v| = 2^-16 it is what keeps the V split's floor
    inside it.
"""
import functools

import pytest
import torch

from tests import att_cases as A
from tests import emul_cabi as E

BAR = A.ATT_EXACT_C[2]
FAULT_FACTOR = 5.0


@functools.lru_cache(maxsize=None)      # every case once, shared by all the tests below
def _contract(name):
    case = next(c for c in A.CASES if c[0] == name)
    qkv, kl = A.make_qkv(case), A.key_lens(case)
    return qkv, kl, *E.attention_contract(qkv, A.H, kl)


def _err(name, p_scale=E.ATT_PSCALE, with_r=True):
    qkv, kl, o64, R = _contract(name)
    got = E.attention_fused_emul(qkv, A.H, kl, p_scale)
    return A.scores(qkv, kl, got, o64, R if with_r else torch.zeros_like(R))


@pytest.mark.parametrize("family", ["plateau", "pfloor"])
def test_unscaled_p_split_exceeds_bar(family):
    errs = {c[0]: _err(c[0], p_scale=1.0)[0] for c in A.CASES if c[1] == family}
    assert max(errs.values()) >= FAULT_FACTOR * BAR, errs


@pytest.mark.parametrize("name", [c[0] for c in A.CASES])
def test_emulated_kernel_within_quarter_bar(name):
    err, _ = _err(name)
    assert err <= BAR / 4, (name, err)


def test_contract_is_the_exact_attention():
    """o64 of attention_contract is E.attention in fp64, padded rows included."""
    qkv, kl, o64, _ = _contract("adv_tied_2^8")
    assert torch.allclose(o64, E.attention(qkv.double(), A.H, kl), rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", ["vscale_2^0", "kqscale_2^0"])
def test_stated_precision_is_a_fraction_of_the_bar(name):
    _, r = _err(name)
    assert r <= BAR / 4, (name, r)


def test_stated_precision_carries_the_v_floor():
    """|v| ~ 2^-16: 16 v has a subnormal lo, so each value carries up to 2^-29 absolute.  Without R the emulated kernel leaves the bar;
    R is larger still and takes it back within a quarter of the bar."""
    err_raw, _ = _err("vscale_2^-16", with_r=False)
    err, r = _err("vscale_2^-16")
    assert err_raw > BAR and r > err_raw and err <= BAR / 4, (err_raw, r, err)
