"""First-contact check of the tensor-core contraction path: the same bf16 batch through the FMA path and the tensor-core
path, teacher-forced, per-block residual and logit differences per step."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from tests.cases import AR_CASES, ar_case_inputs, _unit
from sopro_b200.engine import ArEngine, Sampling

torch.set_grad_enabled(False)
spec = AR_CASES["default_bf16"]
cfg, sd, _ = ar_case_inputs(spec)
eng = ArEngine(cfg, sd, 0, "bf16")
B, steps, L = int(sys.argv[1]) if len(sys.argv) > 1 else 8, int(sys.argv[2]) if len(sys.argv) > 2 else 6, 52
D, NL, V = int(cfg.d_model), int(cfg.n_layers_ar), cfg.ar_vocab()
cond = torch.stack([_unit(steps * D, 7000 + i).view(steps, D) for i in range(B)])
txt = torch.stack([_unit(L * D, 7500 + i).view(L, D) for i in range(B)])
noise = torch.empty(B, steps, 50).exponential_(1.0, generator=torch.Generator().manual_seed(0))
res = {}
for mode in (0, 1):
    ses = eng.session(B, steps, L)
    ses.set_contraction(mode)
    blocks = torch.zeros(steps, NL, B, D, device="cuda")
    logits = torch.zeros(steps, B, V, device="cuda")
    ses.set_trace(blocks, logits)
    ses.begin(cond, txt, [L] * B, noise, Sampling(min_gen_frames=2 ** 31 - 1))
    ses.run()
    torch.cuda.synchronize()
    toks, n, _ = ses.read()
    res[mode] = (blocks.cpu(), logits.cpu(), toks.copy())
    ses.close()
b0, l0, t0 = res[0]
b1, l1, t1 = res[1]
print("tokens equal:", np.array_equal(t0, t1))
for t in range(min(steps, 3)):
    for li in range(NL):
        d = (b0[t, li] - b1[t, li]).abs()
        print(f"step {t} block {li}: max|fma - tc| {float(d.max()):.3e}  (|x| max {float(b0[t, li].abs().max()):.3f}) nan={int(torch.isnan(b1[t, li]).sum())}")
    d = (l0[t] - l1[t]).abs()
    print(f"step {t} logits : max|fma - tc| {float(d.max()):.3e}  (|logit| max {float(l0[t].abs().max()):.3f}) nan={int(torch.isnan(l1[t]).sum())}")
    if t == 0:
        print("  per-utterance logits diff:", [f"{float((l0[0, u] - l1[0, u]).abs().max()):.2e}" for u in range(B)])
print("first tokens fma:", t0[:, :steps].tolist()[:3])
print("first tokens tc :", t1[:, :steps].tolist()[:3])
