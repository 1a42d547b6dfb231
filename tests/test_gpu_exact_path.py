"""GPU: every FastSpeech2 precision policy (fs2_acoustic_model.tc_mask) against the CPU oracle at full batch sizes, with the flip-aware
protocol of tests/test_gpu_model.py.  The default policy is covered there; here the decoder / PostNet on split-FP16 tiles (F8 bits
cleared), on the exact fp32 kernels, and the all-exact model (tc_mask = 0), which is the yardstick the tensor-core paths are measured
against."""
import pytest
import torch

from fastspeech2_b200 import _lib as L
from fastspeech2_b200 import synth
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O
from tests.test_gpu_model import MEL_TOL, _free_running_then_teacher_forced

pytestmark = pytest.mark.gpu
DEV = "cuda"

DEFAULT = L.TC_ENCODER | L.TC_PREDICTORS | L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8
POLICIES = {
    "split3_decoder_postnet": DEFAULT & ~(L.TC_DECODER_F8 | L.TC_POSTNET_F8),
    "exact_decoder_postnet": DEFAULT & ~(L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8),
    "all_exact": 0,
}
# The all-exact model differs from the oracle only in fp32 summation order, so it gets its own mel bar: the largest difference measured
# over CONFIGS on an H100 80GB HBM3 (700 W power limit) was 2.7e-6 (mel and PostNet mel), 4.4x inside this bar and 360x inside MEL_TOL.
EXACT_MEL_TOL = 1.2e-5
CONFIGS = {
    # name: (dataset, weight seed, make_batch arguments)
    "lj_B16_L128": ("LJSpeech", 41, dict(B=16, L=128, seed=42)),
    "libri_configs3_B64": ("LibriTTS", 43, dict(B=64, L=256, seed=44, n_speakers=904, min_len=64)),
    # frame-level pitch / energy predictors on the decoder's rows (B * T frames), raw-valued heads, log-spaced pitch edges
    "lj_paper_B8_L128": ("LJSpeech_paper", 45, dict(B=8, L=128, seed=46)),
}


@pytest.fixture(scope="module")
def oracle_cache():
    """One oracle evaluation per config, free-running and teacher-forced on its own decisions, shared by every policy."""
    return {}


def _oracle(cache, name, scratch):
    if name not in cache:
        from fastspeech2_b200 import configs
        from oracle.gen_golden import paper_state_dict
        dataset, seed, mb = CONFIGS[name]
        mb = dict(mb)
        pc, mc = configs.make_configs(dataset, scratch)
        paper = dataset == "LJSpeech_paper"
        sd = paper_state_dict(pc, mc, seed) if paper else synth.fastspeech2_state_dict(pc, mc, seed=seed)
        kw = dict(pitch_level="frame_level", energy_level="frame_level") if paper else {}
        batch = synth.make_batch(mb.pop("B"), mb.pop("L"), **mb)
        spk, texts, lens, Lm = batch
        ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, **kw)
        ref_tf = O.fastspeech2_forward(sd, spk, texts, lens, Lm, None, ref[9], int(ref[9].max()), ref[2], ref[3], ref[5].long(), **kw)
        cache[name] = ((pc, mc), sd, batch, (ref, ref_tf), paper)
    return cache[name]


@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_precision_policy_vs_oracle(cfg, policy, oracle_cache, scratch, parity_log):
    cfgs, sd, batch, refs, paper = _oracle(oracle_cache, cfg, scratch)
    m = FastSpeech2(*cfgs)
    m.load_state_dict(sd)
    m.tc_mask = POLICIES[policy]
    m = m.to(DEV).eval()
    _free_running_then_teacher_forced(m, sd, batch, f"fs2_policy_{policy}_{cfg}", parity_log, oracle=refs,
                                      mel_tol=EXACT_MEL_TOL if policy == "all_exact" else MEL_TOL, raw_heads=paper)
