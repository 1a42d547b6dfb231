"""CPU emulation of candidate tensor-core operand splits on the HiFi-GAN generator (exact fp64 accumulation of the rounded
operands), against the fp64 oracle.  Decides which split the tensor-core conv kernel may use.

  split3 : a = hi + lo (fp16, fp16), w likewise:  ah*wh + al*wh + ah*wl                 (3 FP16 MMAs, round 1)
  f16f8  : main ah*wh in fp16; correction [al8 | ah8] . [wh8 ; wl8] in e4m3            (1 FP16 + 1 E4M3 MMA)
  f16    : ah*wh only

Usage: python scripts/emul_split_precision.py [--real] [--frames 60]
"""
import argparse
import io
import math
import os
import sys
import zipfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200 import configs, synth  # noqa: E402
from oracle import fs2_oracle as O  # noqa: E402

E4 = torch.float8_e4m3fn
PA_LO, PA_HI = 12, 0          # activation scales: al8 = e4m3(al * 2^12), ah8 = e4m3(ah)


def e4(x):
    return x.clamp(-448.0, 448.0).to(E4).to(torch.float64)


def wscale(w):
    m = float(w.abs().max())
    return 2.0 ** math.floor(math.log2(16384.0 / m))


class Emul:
    def __init__(self, mode):
        self.mode = mode
        self.amax = 0.0

    def operands(self, a, w):
        s = wscale(w)
        ws = (w.double() * s).float()
        wh = ws.half().float()
        wl = (ws - wh)
        a = a.float()
        self.amax = max(self.amax, float(a.abs().max()))
        ah = a.half().float()
        al = a - ah
        return s, ah.double(), al.double(), wh.double(), wl.double()

    def conv(self, fn, a, w, b, **kw):
        """fn(a, w, None, **kw) is linear in both operands."""
        s, ah, al, wh, wl = self.operands(a, w)
        y = fn(ah, wh, None, **kw)
        if self.mode == "split3":
            y = y + fn(al.float().half().double(), wh, None, **kw) + fn(ah, wl.float().half().double(), None, **kw)
        elif self.mode == "f16f8":
            t1 = fn(e4(al * 2.0 ** PA_LO), e4(wh * 2.0 ** -PA_LO), None, **kw)
            t2 = fn(e4(ah * 2.0 ** PA_HI), e4(wl * 2.0 ** -PA_HI), None, **kw)
            y = y + t1 + t2
        elif self.mode == "f16f8_wexact":   # weights' correction in fp8 but activation hi in fp8 -- same thing; placeholder
            raise NotImplementedError
        y = (y / s).float()
        if b is not None:
            y = y + b.float()[None, :, None]
        return y


def hifigan_emul(sd, mel, em, rates=(8, 8, 2, 2), ks=(16, 16, 4, 4), rks=(3, 7, 11), dils=((1, 3, 5),) * 3):
    sd = O.fold_weight_norm(sd) if any(k.endswith(".weight_v") for k in sd) else sd
    nk = len(rks)
    x = em.conv(F.conv1d, mel, sd["conv_pre.weight"], sd["conv_pre.bias"], padding=3)
    for i, (u, k) in enumerate(zip(rates, ks)):
        x = F.leaky_relu(x, 0.1)
        x = em.conv(F.conv_transpose1d, x, sd[f"ups.{i}.weight"], None, stride=u, padding=(k - u) // 2) + sd[f"ups.{i}.bias"][None, :, None]
        acc = None
        for j, (rk, dl) in enumerate(zip(rks, dils)):
            r = x
            p = f"resblocks.{i * nk + j}"
            for m, d in enumerate(dl):
                t = em.conv(F.conv1d, F.leaky_relu(r, 0.1), sd[f"{p}.convs1.{m}.weight"], sd[f"{p}.convs1.{m}.bias"], dilation=d,
                            padding=(rk * d - d) // 2)
                t = em.conv(F.conv1d, F.leaky_relu(t, 0.1), sd[f"{p}.convs2.{m}.weight"], sd[f"{p}.convs2.{m}.bias"], padding=(rk - 1) // 2)
                r = t + r
            acc = r if acc is None else acc + r
        x = acc / nk
    x = F.leaky_relu(x)
    x = F.conv1d(x, sd["conv_post.weight"], sd["conv_post.bias"], padding=3)      # conv_post runs on CUDA cores in fp32
    return torch.tanh(x)


def real_ckpt(name="generator_LJSpeech.pth.tar"):
    z = zipfile.ZipFile(f"/root/reference/hifigan/{name}.zip")
    return torch.load(io.BytesIO(z.read(name)), map_location="cpu")["generator"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    a = ap.parse_args()
    torch.set_num_threads(8)
    mel = synth.make_mel(2, a.frames, seed=3)
    cases = {"synthetic(seed 1)": synth.hifigan_state_dict(configs.HIFIGAN_CONFIG, seed=1),
             "real LJSpeech ckpt": real_ckpt(), "real universal ckpt": real_ckpt("generator_universal.pth.tar")}
    for name, sd in cases.items():
        want64 = O.hifigan_forward(sd, mel, dtype=torch.float64)
        want32 = O.hifigan_forward(sd, mel)
        print(f"== {name}: peak {float(want64.abs().max()):.3f}; fp32 oracle vs fp64 {float((want32.double() - want64).abs().max()):.2e}")
        for mode in ("f16", "f16f8", "split3"):
            em = Emul(mode)
            got = hifigan_emul(sd, mel, em)
            print(f"   {mode:7s}: max-abs vs fp64 {float((got.double() - want64).abs().max()):.2e}   vs fp32 oracle "
                  f"{float((got - want32).abs().max()):.2e}   (max |activation| into a conv {em.amax:.1f})")


if __name__ == "__main__":
    main()
