"""Barrier timeline of one persistent decoder step (BW_MEGA_TRACE=1): per phase, how long the slowest CTA worked and how
long the barrier itself took, and per GEMV phase how long the warps waited for their weight rows after x was staged."""
import os
import sys

import numpy as np
import torch

os.environ["BW_MEGA_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from thewhisper_b200 import synthetic as S  # noqa: E402
from thewhisper_b200.engine import DecodeOptions, ModelDims, WhisperEngine, pack_weights  # noqa: E402
from tools.profile_decode import random_state_dict  # noqa: E402

dev = torch.device("cuda:0")
dims = ModelDims.from_hf_config(S.make_hf_config("large-v3"))
sd = random_state_dict(dims, dev)
w = pack_weights(sd, dims, sd["model.encoder.embed_positions.weight"], dev)
del sd
eng = WhisperEngine({}, dims, chunk_length_s=30, device="cuda:0", max_audios=1, weights=w)
g = S.make_generation_config("large-v3", eos_suppressed=True)
opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens), begin_suppress_tokens=list(g.begin_suppress_tokens))
eng.logmel(S.synth_audio(30, seed=1000)[None])
eng.encode(1)
prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]], dtype=np.int32)
eng.decode_begin(prompt, 1, 1, opts)
eng.decode_run(40)
torch.cuda.synchronize()
N = 264
nsm = torch.cuda.get_device_properties(0).multi_processor_count
raw = eng.buffer("mega_trace", torch.int64, (nsm * N * 6,)).cpu().numpy()
tr = raw[: nsm * N * 2].reshape(nsm, N, 2)
mk = raw[nsm * N * 2:].reshape(nsm, N, 4)
nb = 1 + 8 * dims.dec_layers
arr, rel = tr[:, :nb, 0], tr[:, :nb, 1]
t0 = rel[:, 0].min()
names = ["embed"] + [f"L{l}.{p}" for l in range(dims.dec_layers) for p in ("A qkv", "B self", "C oproj", "D xq", "E cross", "F xo", "G fc1", "H fc2")]
work, barlat = [], []
for b in range(nb):
    start = rel[:, b - 1].min() if b > 0 else arr[:, 0].min() - 1
    work.append(arr[:, b].max() - start)
    barlat.append(rel[:, b].max() - arr[:, b].max())
work, barlat = np.array(work), np.array(barlat)
print("step span (first arrive -> last release): %.1f us" % ((rel[:, nb - 1].max() - arr[:, 0].min()) / 1e3))
print("sum slowest-CTA work %.1f us, sum barrier latency %.1f us" % (work.sum() / 1e3, barlat.sum() / 1e3))
for ph in range(8):
    idx = [1 + 8 * l + ph for l in range(dims.dec_layers)]
    print("%-8s work avg %.2f us (min %.2f max %.2f)   barrier avg %.2f us   spread of arrivals avg %.2f us" % (
        names[1 + ph].split(".")[1], work[idx].mean() / 1e3, work[idx].min() / 1e3, work[idx].max() / 1e3, barlat[idx].mean() / 1e3,
        np.mean([arr[:, i].max() - arr[:, i].min() for i in idx]) / 1e3))
l = 5
for ph in range(8):
    i = 1 + 8 * l + ph
    a = arr[:, i] - (rel[:, i - 1].min())
    print("layer5", names[i], "arrive offsets us: min %.2f med %.2f max %.2f argmax CTA %d" % (a.min() / 1e3, np.median(a) / 1e3, a.max() / 1e3, a.argmax()))

print("marks relative to the release of the previous barrier (median over CTAs / max), layer 5:")
for ph, nm in ((0, "A qkv"), (2, "C oproj"), (3, "D xq"), (6, "G fc1"), (7, "H fc2")):
    i = 1 + 8 * l + ph
    base = rel[:, i - 1]
    out = []
    for j, lab in ((2, "x staged"), (0, "last slab landed"), (3, "warp0 done"), (1, "last warp done")):
        d = (mk[:, i, j] - base) / 1e3
        d = d[mk[:, i, j] > 0]
        out.append("%s %.2f/%.2f" % (lab, np.median(d), d.max()))
    out.append("arrive %.2f/%.2f" % (np.median(arr[:, i] - base) / 1e3, (arr[:, i] - base).max() / 1e3))
    print("  %-8s %s" % (nm, "  ".join(out)))

# slab exposure: how long a CTA's warps waited for their weight rows after x was staged, max(0, last slab landed - x staged)
print("slab exposure per GEMV phase, median / max over CTAs, averaged over the %d layers:" % dims.dec_layers)
tot_med = tot_max = 0.0
for ph, nm in ((0, "A qkv"), (2, "C oproj"), (3, "D xq"), (5, "F xo"), (6, "G fc1"), (7, "H fc2")):
    med, mx = [], []
    for ll in range(dims.dec_layers):
        i = 1 + 8 * ll + ph
        ok = mk[:, i, 0] > 0
        e = np.maximum(0, mk[ok, i, 0] - mk[ok, i, 2]) / 1e3
        med.append(np.median(e))
        mx.append(e.max())
    tot_med += np.sum(med)
    tot_max += np.sum(mx)
    print("  %-8s median %.2f us  max %.2f us" % (nm, np.mean(med), np.mean(mx)))
print("  per step: sum of medians %.1f us, sum of maxima %.1f us" % (tot_med, tot_max))

i = 1 + 8 * l + 4
base = rel[:, i - 1]
busy = mk[:, i, 0] > 0
out = []
for j, lab in enumerate(("K/V + q ready", "scores done", "max known", "PV folded")):
    d = (mk[busy, i, j] - base[busy]) / 1e3
    out.append("%s %.2f/%.2f" % (lab, np.median(d), d.max()))
print("  E cross  " + "  ".join(out))

dns = (mk[busy, i, 1] - mk[busy, i, 0]).astype(np.float64)
dcy = (mk[busy, i, 3] - mk[busy, i, 2]).astype(np.float64)
print("  SM clock during E (cycles / ns between two marks): median %.3f GHz (ns %.0f, cycles %.0f)" % (np.median(dcy / dns), np.median(dns), np.median(dcy)))

end = tr[:, nb, 0]
print("LM head (last barrier release -> CTA done): median %.1f us, max %.1f us" % (np.median(end - rel[:, nb - 1].max()) / 1e3, (end.max() - rel[:, nb - 1].max()) / 1e3))
