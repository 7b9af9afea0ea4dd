"""Per-stage timeline of one AR step from the kernel's own clock64 stamps, with each GEMV stage's warp task shape.
Arguments B:wdtype:team[:shape], shape 0 = the host's choice (default), 1 = always wide, 2 = always narrow."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from tests.cases import AR_CASES, ar_case_inputs, _unit
from sopro_b200.engine import ArEngine, Sampling

torch.set_grad_enabled(False)


def stage_names(cfg, fused):
    names = []
    attn = set(cfg.ar_attn_layers())
    for i in range(int(cfg.n_layers_ar)):
        names += [f"L{i}.glu", f"L{i}.ffn1", f"L{i}.ffn2"]
        if i in attn:
            names += [f"L{i}.qatt", f"L{i}.o"] if fused else [f"L{i}.q", f"L{i}.att", f"L{i}.o"]
    return names + ["head", "sample"]


def run(B, wdtype, team=0, shape=0, steps=64, L=52, step=40):
    spec = AR_CASES["default_bf16" if wdtype == "bf16" else "default_fp32"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = ArEngine(cfg, sd, 0, wdtype)
    D = int(cfg.d_model)
    cond = (_unit(steps * D, 1).view(1, steps, D).expand(B, steps, D) + 0.01 * torch.arange(B).view(B, 1, 1)).contiguous()
    txt = _unit(L * D, 2).view(1, L, D).expand(B, L, D).contiguous()
    noise = torch.empty(B, steps, 50).exponential_(1.0, generator=torch.Generator().manual_seed(0))
    ses = eng.session(B, steps, L)
    if team: ses.set_team(team)
    ses.set_task_shape(shape)
    buf = torch.zeros(eng.num_sms, 224, dtype=torch.int64, device="cuda")
    ses.set_timing(buf, step)
    ses.begin(cond, txt, [L] * B, noise, Sampling(min_gen_frames=2**31 - 1))
    ses.run(); torch.cuda.synchronize()
    t = buf.cpu().numpy()
    # the fused q + attention stage is used when a head's Wq rows fit two ring buffers (batched launches)
    fused = os.environ.get("SOPRO_AR_QATT", "1") != "0" and B >= 8
    names = stage_names(cfg, fused)
    ns = len(names)
    clk = 1.0  # cycles
    shapes = [sh for _k, sh in ses.stage_shapes()]
    print(f"== B={B} {wdtype} team={team} shape mode={shape}: per-stage cycles (median / max over CTAs)")
    tot = np.zeros(5)
    for s_i, nm in enumerate(names):
        base = 1 + 5 * s_i
        t0 = t[:, base - 1]                      # previous release (or step start)
        staged, tiles, done, arr, rel = (t[:, base + k] for k in range(5))
        ok = rel > 0
        parts = [(staged - t0)[ok], (tiles - staged)[ok], (done - tiles)[ok], (arr - done)[ok], (rel - arr)[ok]]
        tot += [np.median(x) for x in parts]
        sh = shapes[s_i] if any(nm.endswith(k) for k in (".glu", ".ffn1", ".ffn2", ".q", ".o", "head")) else ""
        print(f"  {nm:9s} {sh:6s} stage-in {np.median(parts[0]):6.0f}/{parts[0].max():6.0f}  tiles {np.median(parts[1]):6.0f}/{parts[1].max():6.0f}  "
              f"tail {np.median(parts[2]):6.0f}/{parts[2].max():6.0f}  post {np.median(parts[3]):5.0f}  wait {np.median(parts[4]):6.0f}/{parts[4].max():6.0f} (min {parts[4].min():5.0f})")
    sm = t[int(np.argmax(t[:, 161] > 0)), 160:170]  # the CTA that ran a sampler
    print("  sampler phases (CTA 0):", [int(b - a) for a, b in zip(sm[:-1], sm[1:])],
          "= fetch, penalise, max, exp+sum, probs, lower bound, compaction, sort/top-p/draw, bookkeeping")
    span = (t[:, 5 * ns] - t[:, 0])
    print(f"  step span cycles median {np.median(span[span>0]):.0f}; sums of medians stage-in {tot[0]:.0f} tiles {tot[1]:.0f} tail {tot[2]:.0f} post {tot[3]:.0f} wait {tot[4]:.0f}")


if __name__ == "__main__":
    cfgs = [(1, "fp32", 0), (64, "bf16", 0)]
    if len(sys.argv) > 1:  # e.g. 64:bf16:8 1:fp32:0 64:bf16:0:1
        cfgs = [(int(f[0]), f[1], int(f[2]), int(f[3]) if len(f) > 3 else 0) for f in (a.split(":") for a in sys.argv[1:])]
    for c in cfgs:
        run(*c)
