"""CPU: the voices of tests/voice_cases.py and the batches tests/test_gpu_acoustic_voices_plans.py runs them at.
  * the fixture's voices differ in every state tensor a kernel reads, in every tensor-core layer's weight-scale header and in the
    segment headers of every K-segmented conv, and the same checks fail on the plain synthetic seeds;
  * each voice is a sane model on the CPU oracle;
  * on 132 SMs (H100 SXM) the group batches plan the PostNet's first conv at every NG the planner gives it, with a voice mix that
    separates every CTA's consecutive work items, and the exact path's batches reach every (BM, BN) tile the acoustic convs plan."""
import pytest

from fastspeech2_b200 import synth
from tests import voice_cases as V

SMS = 132


def test_fixture_voices_differ_in_every_table_and_header(lj_configs):
    pc, mc = lj_configs
    hdrs = V.check_voices(V.voice_state_dicts(pc, mc), mc)
    seg = [k for k in hdrs[0] if len(hdrs[0][k]) > 1]
    # 4 tensor-core layers per FFT block, the predictors' 6 convs, mel_linear and 5 PostNet convs; more than one segment: the encoder's
    # FFN convs (9 taps, 4 x 256 channels) and the predictor convs (3 taps)
    assert len(hdrs[0]) == 4 * 4 + 6 * 4 + 3 * 2 + 1 + 5 and len(seg) == 4 * 2 + 3 * 2, sorted(seg)


def test_fixture_checks_fail_on_the_plain_seeds(lj_configs):
    """The checks see what synthetic seeds share: position tables, duration bias and bins, and the headers."""
    pc, mc = lj_configs
    plain = [synth.fastspeech2_state_dict(pc, mc, seed=s) for s in (51, 52, 53)]
    for k in ("variance_adaptor.pitch_bins", "variance_adaptor.energy_bins"):
        plain[2][k] = plain[2][k] * 1.07
    with pytest.raises(AssertionError, match="position_enc"):
        V.check_state(plain)
    with pytest.raises(AssertionError, match="shared between voices"):
        V.check_headers(plain, mc)


def test_fixture_voices_are_sane(lj_configs):
    pc, mc = lj_configs
    V.check_sane(V.voice_state_dicts(pc, mc), pc, mc)


@pytest.mark.parametrize("target", V.GROUP_TARGETS, ids=lambda t: f"{t[0]}_ng{t[2]}")
def test_group_batches_plan_their_ng(target):
    mask, fmt, NG, T = target
    B, p, fb, voice = V.group_batch(fmt, NG, T, SMS)
    assert p["NG"] == NG and p["grid"] == SMS, p
    assert sorted(set(voice)) == list(range(V.MAX_VOICES)) and len(voice) == B
    groups = p["n_items"] // NG // (B * p["tiles_per_batch"])
    for rows in (None, fb[4]):
        assert V.clashes(voice, V.items(B, rows, T, groups), p["grid"]) == 0
    assert int(fb[4].max()) == T and B * T <= 64 * 2048, (B, T)


def test_group_targets_cover_every_ng_of_the_postnet():
    """Every NG > 1 the planner gives the PostNet's first conv at batches of up to 64 x 2048 rows, in both formats, is a target."""
    from tests import conv_group_cases as G
    seen = set()
    for fmt in ("f8", "split3"):
        for B in range(1, 65):
            for T in (256, 512, 1012, 2006, 2048):
                ng = G.plan(V.postnet0_case(fmt, 1, T), B, SMS)["NG"]
                if ng > 1:
                    seen.add((fmt, ng))
    assert seen == {(fmt, ng) for _, fmt, ng, _ in V.GROUP_TARGETS}, seen


def test_exact_shapes_reach_every_simt_tile(lj_configs):
    _, mc = lj_configs
    want = V.simt_universe(mc, SMS)
    assert want == {(64, 64), (64, 128), (128, 128)}, want
    assert V.simt_tiles(V.EXACT_SHAPES, mc, SMS) == want
