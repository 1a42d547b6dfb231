"""Decision-flip census (SURVEY.md section 7, hard part 2; VERDICT r01 item 6): durations round(exp(logd) - 1) and the pitch / energy
buckets are discrete, so fp32-level differences can flip them.  For >= 10k phonemes per config this counts, against the CPU oracle,
the flips of (a) the exact fp32 CUDA-core encoder + predictors and (b) the tensor-core three-MMA-split encoder + predictors, with the
distance of every flipped value to its decision boundary.  One JSON line per (config, path).  Usage: python scripts/flip_census.py [seeds]"""
import json, os, sys, tempfile
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200 import configs, synth, _lib as L
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O

DEV = "cuda"
seeds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
torch.set_num_threads(16)
base = L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8
for ds, nspk, Lmax, minlen in (("LJSpeech", 1, 128, None), ("LibriTTS", 904, 192, 64)):
    pc, mc = configs.make_configs(ds, tempfile.mkdtemp())
    for path, mask in (("fp32_cuda_cores", base), ("tensor_core_k_segmented", base | L.TC_ENCODER | L.TC_PREDICTORS)):
        tot = {"config": ds, "encoder_predictors": path, "phonemes": 0, "duration_flips": 0, "pitch_bucket_flips": 0, "energy_bucket_flips": 0,
               "max_err_logd": 0.0, "max_err_pitch": 0.0, "max_err_energy": 0.0, "flip_margins": []}
        for seed in range(seeds):
            sd = synth.fastspeech2_state_dict(pc, mc, seed=50 + seed)
            m = FastSpeech2(pc, mc); m.load_state_dict(sd); m.tc_mask = mask; m = m.to(DEV).eval()
            spk, texts, lens, Lm = synth.make_batch(64, Lmax, seed=60 + seed, n_speakers=nspk, min_len=minlen)
            out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
            p, e, logd, d = O.fastspeech2_decisions(sd, spk, texts, lens, Lm)
            valid = torch.arange(Lm)[None, :] < lens[:, None]
            tot["phonemes"] += int(valid.sum())
            gp, ge, gl, gd = out[2].cpu(), out[3].cpu(), out[4].cpu(), out[5].cpu()
            tot["max_err_logd"] = max(tot["max_err_logd"], float((gl - logd).abs().max()))
            tot["max_err_pitch"] = max(tot["max_err_pitch"], float((gp - p).abs().max()))
            tot["max_err_energy"] = max(tot["max_err_energy"], float((ge - e).abs().max()))
            for b, l in ((gd != d) & valid).nonzero().tolist():
                v = float(torch.exp(logd[b, l].double()) - 1)
                tot["duration_flips"] += 1
                tot["flip_margins"].append(("duration", abs(v - (int(v) + 0.5))))
            for nm, g, r, key in (("pitch", gp, p, "pitch_bucket_flips"), ("energy", ge, e, "energy_bucket_flips")):
                edges = sd[f"variance_adaptor.{nm}_bins"]
                for b, l in ((torch.bucketize(g, edges) != torch.bucketize(r, edges)) & valid).nonzero().tolist():
                    tot[key] += 1
                    tot["flip_margins"].append((nm, float((edges - r[b, l]).abs().min())))
            del m
        print(json.dumps(tot), flush=True)
