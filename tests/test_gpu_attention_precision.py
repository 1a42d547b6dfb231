"""GPU: fs2_attention, both backends, against fp64 across the magnitude cases of tests/att_cases.py: per row,
|o - o64| - R <= ATT_EXACT_C[backend] 2^-24 max|v| (1 + scale max sum|q||k|), with R the fused kernel's stated operand precision
(tests/emul_cabi.py::attention_contract) and R = 0 for the exact kernel, whose operands are fp32."""
import functools

import pytest
import torch

from fastspeech2_b200 import ops
from tests import att_cases as A
from tests import emul_cabi as E

pytestmark = pytest.mark.gpu
DEV = "cuda"


@functools.lru_cache(maxsize=2)
def _contract(name):
    case = next(c for c in A.CASES if c[0] == name)
    qkv, kl = A.make_qkv(case), A.key_lens(case)
    return qkv, kl, *E.attention_contract(qkv, A.H, kl)


# Known failures on the plateau rows, in the bar's units, measured on an H100 80GB HBM3 (700 W) at 300 / 1012 / 4200 keys:
#   fused kernel, 39 / 132 / 629, with and without AF_PSCALE: its tensor cores align each product to the fp32 accumulator and truncate
#     it, so n - 1 equal products lose the same bits n - 1 times and the loss grows with the accumulator's running size, which its bar
#     does not carry (the convolutions' bar does, as accumulator mass).  The pfloor rows, whose accumulator stays small, pass.
#   exact kernel, 2.6 / 2.6 / 3.6 (23 / 71 / 303 before its O and l sums were compensated): what is left is the fp32 rounding of
#     the one dot product per score, which a plateau row turns into the same weight error on every plateau key; the same 2.6 on the
#     127- to 129-key utterances shows that it does not grow with n.
# Strict, so that these cases fail this marker once either kernel is brought inside its bar.
PLATEAU_XFAIL = {
    2: pytest.mark.xfail(strict=True, reason="tensor-core truncation of n equal products adds up n times"),
    0: pytest.mark.xfail(strict=True, reason="fp32 score rounding on a plateau moves every plateau weight alike"),
}


def _params():
    out = []
    for name, fam, *_ in A.CASES:
        for backend in (0, 2):
            marks = [PLATEAU_XFAIL[backend]] if fam == "plateau" else []
            out.append(pytest.param(name, backend, marks=marks, id=f"{name}-{backend}"))
    return out


@pytest.mark.parametrize("name,backend", _params())
def test_attention_magnitudes(name, backend, parity_log):
    qkv, kl, o64, R = _contract(name)
    got = ops.attention(qkv.to(DEV), A.H, kl.to(DEV), backend=backend).cpu()
    assert torch.isfinite(got).all()
    for b, n in enumerate(kl.tolist()):                  # padded query rows are exact zeros
        assert (got[b, max(n, 0):] == 0).all()
    err, r = A.scores(qkv, kl, got, o64, R if backend == 2 else torch.zeros_like(R))
    bar = A.ATT_EXACT_C[backend]
    parity_log("test_attention_magnitudes", case=name, backend=backend, err=err, bar=bar, R_max=r)
    assert err <= bar, (name, backend, err)
