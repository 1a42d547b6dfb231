"""GPU: every fused ResBlock stage of V1 and V2 run as the planner's fs2_resstack launches (fs2_vocoder_resblock_runs) is bit for bit
the whole-group launch, padded and ragged, on the Generator's packed weights -- so the plan changes no output of forward, stream or
stream_pool."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, synth
from fastspeech2_b200.hifigan import AttrDict, Generator

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rows_per_frame(m, i):
    scale = 1
    for u in range(i + 1):
        scale *= m.rates[u]
    return scale


def run_stage(m, pk, i, x, lens, runs, bufs=None):
    """Stage i's ResBlock group on x [B][N][C] issued as `runs` [(j, d0, d1)] (j = -1: the whole group), with the buffers and
    arguments fs2_vocoder_forward uses (model.cu's window_walk over [0, T)); bufs: (y, r1, r2) like x, or None for fresh NaN-filled
    ones.  Returns y.  (scripts/resblock_runs_bench.py times stages through this too.)"""
    nk, nd, scale = m.n_kernels, m.n_dil, _rows_per_frame(m, i)
    ks = [m.rb_k[j] for j in range(nk)]
    dils = [[m.rb_dil[j][d] for d in range(nd)] for j in range(nk)]
    w = lambda name: [[pk[f"rb.{i * nk + j}.{d}.{name}"] for d in range(nd)] for j in range(nk)]
    t1, b1, t2, b2 = w("w1_tc"), w("b1"), w("w2_tc"), w("b2")
    y, r1, r2 = bufs if bufs is not None else (torch.full_like(x, float("nan")) for _ in range(3))
    r = x
    for j, d0, d1 in runs:
        if j < 0:
            ops.resstack(x, ks, dils, t1, b1, t2, b2, out=y, lens=lens, lens_scale=scale)
            continue
        last = d1 == nd
        if d0 == 0:
            r = x
        dst = y if last else (r2 if r is r1 else r1)
        cut = lambda t: [t[j][d0:d1]]
        ops.resstack(r, [ks[j]], [dils[j][d0:d1]], cut(t1), cut(b1), cut(t2), cut(b2), alpha=1.0 / nk if last else 1.0,
                     accumulate=last and j > 0, out=dst, lens=lens, lens_scale=scale)
        r = dst
    return y


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_planned_runs_equal_the_group_launch(cfg, ragged):
    h = AttrDict(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=2))
    gen = gen.eval().to(DEV)
    m, pk, _, _ = gen._pack()
    B, T = 3, 37
    lens = torch.tensor([T, 23, 5], dtype=torch.int32, device=DEV) if ragged else None
    g = torch.Generator().manual_seed(7)
    stages = [i for i in range(m.n_stages) if (m.fused_mask >> i) & 1]
    assert stages == ([2, 3] if cfg == "v1" else [0, 1, 2, 3])
    for i in stages:
        runs = [(r.j, r.d0, r.d1) for r in L.vocoder_resblock_runs(m, i)]
        assert runs and runs[0][0] >= 0, runs          # the planner cuts every fused stage of V1 and V2 into ResBlock runs
        scale = _rows_per_frame(m, i)
        x = (0.7 * torch.randn(B, T * scale, m.c0 >> (i + 1), generator=g)).to(DEV)
        want = run_stage(m, pk, i, x, lens, [(-1, 0, m.n_dil)])
        got = run_stage(m, pk, i, x, lens, runs)
        torch.cuda.synchronize()
        if ragged:
            for b in range(B):
                n = int(lens[b]) * scale
                assert torch.equal(got[b, :n], want[b, :n]), (cfg, i, b)
        else:
            assert torch.isfinite(got).all() and torch.equal(got, want), (cfg, i)
