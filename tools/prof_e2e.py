"""Phase timing of the host-side pipeline around the two CUDA engines (TTFA and synthesize_batch breakdown)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from sopro_b200 import SoproTTS
from sopro_b200.config import SoproTTSConfig
from sopro_b200.tokenizer import IdsTokenizer
from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

dev = torch.device("cuda:0")
cfg = SoproTTSConfig()
tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(), device=str(dev))
ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
text = " ".join(str(17 * i + 5) for i in range(50))


def timed(fn, n=10, warm=3):
    ts = []
    for i in range(n + warm):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        if i >= warm:
            ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, r


with torch.inference_mode():
    t, ids = timed(lambda: tts.encode_text(text))
    print(f"encode_text            {t:8.3f} ms")
    t, prep = timed(lambda: tts.model.prepare_conditioning(ids, ref, max_frames=400, style_strength=cfg.style_strength))
    print(f"prepare_conditioning   {t:8.3f} ms")

    def ar6():
        out = []
        for _t, tok, e in tts.model.ar_stream(prep, max_frames=400, launch_frames=6, seed=1, min_gen_frames=10 ** 9):
            out.append(tok)
            if len(out) == 6:
                break
        return out
    t, h = timed(ar6)
    print(f"ar_stream first 6      {t:8.3f} ms")
    toks = torch.as_tensor(h, device=dev, dtype=torch.long).unsqueeze(0)
    t, win = timed(lambda: tts.model.nar_refine(prep["cond_ar"][:, :6], toks))
    print(f"nar_refine T=6         {t:8.3f} ms")
    t, _ = timed(lambda: tts.codec.decode_full(win.squeeze(0)))
    print(f"mimi decode T=6        {t:8.3f} ms")
    toks400 = torch.randint(0, 2048, (1, 401), device=dev)
    t, w400 = timed(lambda: tts.model.nar_refine(prep["cond_ar"][:, :401], toks400), n=5)
    print(f"nar_refine T=401 B=1   {t:8.3f} ms")
    c64 = prep["cond_ar"][:, :401].expand(64, -1, -1).contiguous()
    t, w = timed(lambda: tts.model.nar_refine(c64, toks400.expand(64, -1).contiguous()), n=3, warm=1)
    print(f"nar_refine T=401 B=64  {t:8.3f} ms")
    t, _ = timed(lambda: tts.codec.decode_full(w400.squeeze(0)), n=5)
    print(f"mimi decode T=401 B=1  {t:8.3f} ms")
    codes = w.permute(0, 2, 1).contiguous()
    t, _ = timed(lambda: tts.codec.engine.decode(codes), n=3, warm=1)
    print(f"mimi decode T=401 B=64 {t:8.3f} ms")
    t, _ = timed(lambda: next(iter(tts.stream(text, ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9))), n=10)
    print(f"stream first chunk     {t:8.3f} ms")
    # steady-state streaming chunk: NAR over ctx + chunk frames, Mimi stream step of one chunk
    ctx = tts.model.rf_nar()
    n = ctx + 6
    toksw = torch.randint(0, 2048, (1, n), device=dev)
    t, winw = timed(lambda: tts.model.nar_refine(prep["cond_ar"][:, :n], toksw), n=5)
    print(f"nar_refine T={n} B=1   {t:8.3f} ms")
    from sopro_b200.codec import MimiStreamDecoder
    msd = MimiStreamDecoder(tts.codec, max_chunk_frames=16)
    st = msd.new_state()
    ts = []
    for i in range(40):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        wv, st = msd.decode_step(winw.squeeze(0)[i * 4 % 100:i * 4 % 100 + 6], st)
        torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    print(f"mimi stream step 6 fr  {np.median(ts[5:]) * 1e3:8.3f} ms")
    msd.release(st)
    t, _ = timed(lambda: sum(1 for _ in tts.stream(text, ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9)), n=3, warm=1)
    print(f"stream 400 frames      {t:8.3f} ms")
    # synthesize_batch(64) phases
    texts = [" ".join(str((17 * i + 5 + 31 * j) % 1000) for i in range(50)) for j in range(64)]
    ids64 = [tts.encode_text(x) for x in texts]
    t, _ = timed(lambda: tts.model.prefill.run(ids64, ref, n_frames=401, style_strength=cfg.style_strength), n=3, warm=1)
    print(f"prefill batch 64       {t:8.3f} ms")
    from sopro_b200.sampling import TapeFeed

    def draw_tapes():
        with TapeFeed(64, 401, cfg.ar_vocab(), 50, dev, list(range(64))) as feed:
            feed.fill(401)
    t, _ = timed(draw_tapes, n=3, warm=1)
    print(f"draw+upload 64 tapes   {t:8.3f} ms")
    t, _ = timed(lambda: tts.synthesize_batch(texts, ref=ref, max_frames=400, seeds=list(range(64)), min_gen_frames=10 ** 9), n=3, warm=1)
    print(f"synthesize_batch(64)   {t:8.3f} ms")
