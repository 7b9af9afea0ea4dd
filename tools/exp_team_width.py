import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tests.cases import AR_CASES, ar_case_inputs, _unit
from sopro_b200.engine import ArEngine, Sampling
torch.set_grad_enabled(False)
spec = AR_CASES["default_bf16"]; cfg, sd, _ = ar_case_inputs(spec)
eng = ArEngine(cfg, sd, 0, "bf16")
D = int(cfg.d_model); steps, L = 401, 52
for B in (1, 2, 4, 8):
    cond = torch.stack([_unit(steps * D, 7000 + i).view(steps, D) for i in range(B)]).cuda()
    txt = torch.stack([_unit(L * D, 7500 + i).view(L, D) for i in range(B)]).cuda()
    noise = torch.empty(B, steps, 50).exponential_(1.0, generator=torch.Generator().manual_seed(0)).cuda()
    ses = eng.session(B, steps, L)
    for _ in range(2):
        ses.begin(cond, txt, [L] * B, noise, Sampling(min_gen_frames=2**31 - 1)); ses.run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(3):
        ses.begin(cond, txt, [L] * B, noise, Sampling(min_gen_frames=2**31 - 1))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ses.run(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    print(f"MAX_P={os.environ.get('SOPRO_AR_MAX_P','-')} B={B}: {min(ts) / steps * 1e3:.1f} us/step", flush=True)
    ses.close()
