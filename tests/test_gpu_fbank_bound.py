"""Every element of the log-fbank front-end on the GPU against the fp64 stage-by-stage reference, within the bound
derived from the kernel's arithmetic (tests/fbank_bound.py; the gate's self-test on an fp32 emulation with seeded
defects is tests/test_fbank_bound_host.py).

Per sample rate, one batched call of about 36 utterances (``fbank_bound.batch``: the edge lengths each followed by a
loud neighbour, frame counts 0 .. 3 mod 4, every signal class, 100 003 samples, and at 16 kHz 2^24 + 12 345 samples)
for each of the four use_logscale x subtract_mean combinations, and ``mk_mfb_batch_vad`` for the energies.  Each
utterance is gated on its own:
  mel        linear, un-subtracted outputs vs m within B (eps where m^ == 0);
  log        log outputs vs the widened dB interval of [m - B, m + B];
  mean_lin / mean_log   mean-subtracted outputs vs the engine's own un-subtracted output;
  energy     the frame energies;
  power_iso  the filters that are one bin of weight 1.0, vs that bin's power and the per-bin power bound.
The max err/bound of each stage, rate and signal class is printed (run with -s)."""
import numpy as np
import pytest
import torch

from deepspeaker_pytorch_b200 import frontend as F
from tests import fbank_bound as FB

pytestmark = pytest.mark.gpu

RATES = (8000, 16000, 11025, 12000, 20499, 50, 100)
STAGES = ("mel", "log", "mean_lin", "mean_log", "energy", "power_iso")


def _split(t, foff):
    a = t.cpu().numpy()
    return [a[foff[u]:foff[u + 1]] for u in range(len(foff) - 1)]


@pytest.mark.parametrize("sr", RATES)
def test_every_element_within_the_derived_bound(cuda_dev, sr):
    utts = FB.batch(sr, seed=sr)
    lens = [x.size for _, x in utts]
    audio = torch.from_numpy(np.concatenate([x for _, x in utts])).to(cuda_dev)
    out = {}
    for log in (False, True):
        for sub in (False, True):
            feats, foff = F.mk_mfb_batch(audio, lens, sr, log, sub)
            foff = foff.numpy()
            out[log, sub] = _split(feats, foff)
    _, foff_v, energy, _ = F.mk_mfb_batch_vad(audio, lens, sr)
    assert np.array_equal(foff_v.numpy(), foff)
    energy = _split(energy, foff)
    torch.cuda.synchronize()
    worst = {}
    for u, (cls, x) in enumerate(utts):
        assert foff[u + 1] - foff[u] == FB.num_frames(x.size, sr)
        R = FB.Reference(x, sr)
        lin, lg = out[False, False][u], out[True, False][u]
        for stage, r in (("mel", FB.mel_ratio(lin, R)), ("log", FB.log_ratio(lg, R)),
                         ("mean_lin", FB.mean_ratio(out[False, True][u], lin)),
                         ("mean_log", FB.mean_ratio(out[True, True][u], lg)),
                         ("energy", FB.energy_ratio(energy[u], R)), ("power_iso", FB.iso_ratio(lin, R))):
            if r.size:
                v = float(np.nan_to_num(r, nan=np.inf).max())
                worst[stage, cls] = max(worst.get((stage, cls), 0.0), v)
    classes = sorted({c for _, c in worst})
    print(f"\nfbank at {sr} Hz, max err/bound per stage and signal class ({len(utts)} utterances, "
          f"{int(foff[-1])} frames, {len(FB.isolated_filters(sr))} isolated filters)")
    print(f"{'class':>16} " + " ".join(f"{s:>9}" for s in STAGES))
    for c in classes:
        print(f"{c:>16} " + " ".join(f"{worst[s, c]:9.3g}" if (s, c) in worst else f"{'-':>9}" for s in STAGES))
    print(f"{'all':>16} " + " ".join(f"{max((v for (s2, _), v in worst.items() if s2 == s), default=0):9.3g}"
                                     for s in STAGES))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad
