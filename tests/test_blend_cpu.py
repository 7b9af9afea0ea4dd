"""Voice blends on the host (sopro_b200/voices.py::blend, segment_table) and the float64 blend oracle
(oracle/blend_oracle.py): construction, flattening, merging, normalisation, every refusal, pickling.  No device."""
import math
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.cases import e2e_inputs

torch.set_grad_enabled(False)
_S = {}


def _geom():
    from sopro_b200 import voices

    return voices.geometry(e2e_inputs()[0])


def _voice(Tr, seed):
    from sopro_b200 import prefill as P

    key = (Tr, seed)
    if key not in _S:
        cfg, sd, _ = e2e_inputs()
        tok = torch.randint(0, 2048, (Tr, 32), generator=torch.Generator().manual_seed(seed))
        _S[key] = P.prepare_reference(sd, cfg, tok, torch.device("cpu"))
    return _S[key]


def _blend(vs, weights=None):
    from sopro_b200 import voices

    return voices.blend(vs, weights, device="cpu", **_geom())


def _sv_mix(svs, ws):
    m = (torch.tensor(ws, dtype=torch.float64)[:, None] * torch.stack([s.double().reshape(-1) for s in svs])).sum(dim=0)
    return (m / float(m.norm())).float().reshape(1, -1)


def test_two_voices_concatenate_frames_and_normalise_weights():
    from sopro_b200.prefill import PreparedReference
    from sopro_b200.voices import VoiceBlend

    a, b = _voice(5, 1), _voice(9, 2)
    m = _blend([a, b], [1.0, 3.0])
    assert isinstance(m, VoiceBlend) and isinstance(m, PreparedReference)
    assert m.segments == (5, 9) and m.weights == (0.25, 0.75)
    assert all(isinstance(w, float) for w in m.weights) and all(isinstance(n, int) for n in m.segments)
    for i in range(3):
        for t in ("k", "v"):
            assert torch.equal(m.ref_kv_caches[i][t], torch.cat([a.ref_kv_caches[i][t], b.ref_kv_caches[i][t]], dim=2))
        assert m.ref_kv_caches[i]["key_padding_mask"] is None
    assert torch.equal(m.ref_seq, torch.cat([a.ref_seq, b.ref_seq], dim=1))
    assert torch.equal(m.ref_tokens_btq, torch.cat([a.ref_tokens_btq, b.ref_tokens_btq], dim=1))
    assert torch.equal(m.sv_ref, _sv_mix([a.sv_ref, b.sv_ref], m.weights)) and m.sv_ref.shape == (1, 192)
    assert abs(float(m.sv_ref.norm()) - 1.0) < 1e-6
    from sopro_b200 import voices

    assert voices.check_voice(m, **_geom()) == 14
    assert _blend([a, b]).weights == (0.5, 0.5)  # None: equal weights


def test_weights_normalise_in_float64_and_round_once_to_float32():
    a, b, c = _voice(5, 1), _voice(9, 2), _voice(3, 3)
    ws = [0.1, 0.7, 1e-3]
    m = _blend([a, b, c], ws)
    tot = math.fsum(ws)
    assert m.weights == tuple(float(np.float32(w / tot)) for w in ws)
    m2 = _blend((a, b, c), tuple(np.float64(w) for w in ws))  # any real numbers, in any sequence
    assert m2.weights == m.weights and torch.equal(m2.sv_ref, m.sv_ref)
    assert _blend([a, b], [2, 6]).weights == _blend([a, b], [np.float32(1), np.int64(3)]).weights == (0.25, 0.75)


def test_one_component_passes_its_voice_through_unchanged():
    a, b = _voice(5, 1), _voice(9, 2)
    for m in (_blend([a]), _blend([a, a]), _blend([a, a], [0.3, 4.0])):
        assert m.segments == (5,) and m.weights == (1.0,)
        assert torch.equal(m.sv_ref, a.sv_ref) and m.sv_ref is not a.sv_ref
        assert all(torch.equal(m.ref_kv_caches[i]["k"], a.ref_kv_caches[i]["k"]) for i in range(3))
        assert torch.equal(m.ref_seq, a.ref_seq)
    # a blend of one blend-segment keeps it too
    mm = _blend([_blend([b])])
    assert mm.segments == (9,) and mm.weights == (1.0,) and torch.equal(mm.sv_ref, b.sv_ref)


def test_repeated_objects_merge_with_their_weights_summed():
    a, b = _voice(5, 1), _voice(9, 2)
    m = _blend([a, b, a], [1.0, 1.0, 2.0])
    assert m.segments == (5, 9) and m.weights == (0.75, 0.25)
    assert torch.equal(m.ref_seq, _blend([a, b], [3.0, 1.0]).ref_seq)
    assert torch.equal(m.sv_ref, _blend([a, b], [3.0, 1.0]).sv_ref)
    # two equal voices prepared separately are two objects, so two segments
    a2 = _voice(5, 1)
    from sopro_b200 import prefill as P

    a3 = P.PreparedReference(a2.ref_tokens_btq, a2.sv_ref.clone(), a2.ref_seq, a2.ref_kv_caches)
    assert _blend([a, a3]).segments == (5, 5)


def test_a_blend_flattens_into_its_segments_with_scaled_weights():
    a, b, c = _voice(5, 1), _voice(9, 2), _voice(3, 3)
    inner = _blend([a, b])
    m = _blend([inner, c])
    assert m.segments == (5, 9, 3) and m.weights == (0.25, 0.25, 0.5)
    flat = _blend([a, b, c], [1.0, 1.0, 2.0])
    assert flat.segments == m.segments and flat.weights == m.weights
    assert torch.equal(m.sv_ref, flat.sv_ref) and torch.equal(m.segment_sv, flat.segment_sv)
    for i in range(3):
        assert torch.equal(m.ref_kv_caches[i]["v"], flat.ref_kv_caches[i]["v"])
    assert torch.equal(m.ref_tokens_btq, flat.ref_tokens_btq)
    # the same blend twice merges segment by segment; a blend and a plain voice it was built from do not (no references)
    assert _blend([inner, inner]).segments == (5, 9)
    assert _blend([inner, a]).segments == (5, 9, 5)
    # the blend holds no reference to its components
    assert all(t is not a.ref_kv_caches[0]["k"] for t in (m.ref_kv_caches[0]["k"],))


def test_pickle_round_trip():
    from sopro_b200.voices import VoiceBlend

    m = _blend([_voice(5, 1), _voice(9, 2)], [2.0, 1.0])
    r = pickle.loads(pickle.dumps(m))
    assert type(r) is VoiceBlend and r.segments == m.segments and r.weights == m.weights
    assert torch.equal(r.sv_ref, m.sv_ref) and torch.equal(r.ref_seq, m.ref_seq) and torch.equal(r.segment_sv, m.segment_sv)
    assert all(torch.equal(r.ref_kv_caches[i][t], m.ref_kv_caches[i][t]) for i in range(3) for t in ("k", "v"))


def test_segment_table():
    from sopro_b200 import voices

    a, b, c = _voice(5, 1), _voice(9, 2), _voice(3, 3)
    m = _blend([a, b, c], [1.0, 2.0, 1.0])
    n_seg, frames, ws = voices.segment_table([a, m, b], [5, 17, 9])
    assert n_seg == [1, 3, 1] and frames == [5, 5, 9, 3, 9] and ws == [1.0, 0.25, 0.5, 0.25, 1.0]
    with pytest.raises(ValueError):
        voices.segment_table([m], [16])


def _bad_geometry():
    from sopro_b200 import prefill as P

    a = _voice(5, 1)
    return P.PreparedReference(a.ref_tokens_btq, a.sv_ref, a.ref_seq, a.ref_kv_caches[:2])


def _two_rows():
    from sopro_b200 import prefill as P

    a = _voice(5, 1)
    return P.PreparedReference(a.ref_tokens_btq, torch.cat([a.sv_ref, a.sv_ref]), a.ref_seq, a.ref_kv_caches)


def _opposed():
    from sopro_b200 import prefill as P

    a = _voice(5, 1)
    return [a, P.PreparedReference(a.ref_tokens_btq, -a.sv_ref, a.ref_seq, a.ref_kv_caches)]


def _long(n):
    return [_voice(2048, 10 + i) for i in range(n)]


REFUSALS = [
    ("not a sequence", lambda: (_voice(5, 1), None), TypeError),
    ("a string", lambda: ("ab", None), TypeError),
    ("not a voice", lambda: ([_voice(5, 1), "b"], None), TypeError),
    ("a tensor as a voice", lambda: ([_voice(5, 1).sv_ref], None), TypeError),
    ("empty", lambda: ([], None), ValueError),
    ("17 segments", lambda: ([_voice(1, 100 + i) for i in range(17)], None), ValueError),
    ("17 segments after flattening", lambda: ([_blend([_voice(1, 100 + i) for i in range(16)]), _voice(1, 200)], None), ValueError),
    ("short weights", lambda: ([_voice(5, 1), _voice(9, 2)], [1.0]), ValueError),
    ("long weights", lambda: ([_voice(5, 1), _voice(9, 2)], [1.0, 1.0, 1.0]), ValueError),
    ("weights a string", lambda: ([_voice(5, 1)], "1"), TypeError),
    ("weights a number", lambda: ([_voice(5, 1)], 1.0), TypeError),
    ("weights a tensor", lambda: ([_voice(5, 1)], torch.ones(1)), TypeError),
    ("a bool weight", lambda: ([_voice(5, 1), _voice(9, 2)], [True, 1.0]), TypeError),
    ("a string weight", lambda: ([_voice(5, 1), _voice(9, 2)], ["1", 1.0]), TypeError),
    ("a nan weight", lambda: ([_voice(5, 1), _voice(9, 2)], [float("nan"), 1.0]), ValueError),
    ("an inf weight", lambda: ([_voice(5, 1), _voice(9, 2)], [float("inf"), 1.0]), ValueError),
    ("a zero weight", lambda: ([_voice(5, 1), _voice(9, 2)], [0.0, 1.0]), ValueError),
    ("a negative weight", lambda: ([_voice(5, 1), _voice(9, 2)], [-1.0, 1.0]), ValueError),
    ("wrong geometry", lambda: ([_voice(5, 1), _bad_geometry()], None), ValueError),
    ("two speaker vectors", lambda: ([_voice(5, 1), _two_rows()], None), ValueError),
    ("4097 frames", lambda: (_long(2) + [_voice(1, 300)], None), ValueError),
    ("speaker vectors that cancel", lambda: (_opposed(), None), ValueError),
]


@pytest.mark.parametrize("name,make,exc", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_leave_the_global_generator_untouched(name, make, exc):
    vs, ws = make()
    state = torch.get_rng_state()
    with pytest.raises(exc):
        _blend(vs, ws)
    assert torch.equal(torch.get_rng_state(), state)


def test_4096_frames_and_16_segments_are_accepted():
    m = _blend(_long(2))
    assert sum(m.segments) == 4096
    m = _blend([_voice(1, 100 + i) for i in range(16)])
    assert m.segments == (1,) * 16 and len(m.weights) == 16


# ---------------------------------------------------------------------------------------------------------------
# the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
def _pos():
    from sopro_b200 import prefill as P

    cfg = e2e_inputs()[0]
    return (P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), "cpu"),
            P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), "cpu"))


def test_oracle_of_one_segment_equals_prepare_conditioning():
    from oracle import blend_oracle as BO
    from sopro_b200 import prefill as P

    cfg, sd, inp = e2e_inputs()
    tpos, fpos = _pos()
    a = _voice(38, 4)
    kw = dict(max_frames=20, style_strength=1.2, text_pos=tpos, frame_pos=fpos)
    ids = inp["text_ids"]
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    a64 = P.PreparedReference(a.ref_tokens_btq, a.sv_ref.double(), a.ref_seq.double(),
                              [{k: (t.double() if isinstance(t, torch.Tensor) else t) for k, t in c.items()} for c in a.ref_kv_caches])
    want = P.prepare_conditioning(sd64, cfg, ids, a64, device="cpu", **kw)
    got = BO.prepare_conditioning(sd, cfg, ids, _blend([a]), **kw)
    plain = BO.prepare_conditioning(sd, cfg, ids, a, **kw)
    assert torch.equal(got["cond_ar"], plain["cond_ar"]) and got["cond_ar"].dtype == torch.float64
    # prefill.ref_xattn attends in float32: equal to that rounding
    assert float((got["cond_ar"] - want["cond_ar"]).abs().max()) < 1e-5
    assert float((got["txt_seq"] - want["txt_seq"]).abs().max()) == 0.0


def test_oracle_mixed_readout_is_the_weighted_sum_of_per_voice_readouts():
    from oracle import blend_oracle as BO

    g = torch.Generator().manual_seed(3)
    q = torch.randn(2, 2, 7, 16, generator=g, dtype=torch.float64)
    frames, ws = [3, 1, 12], [0.25, 0.5, 0.25]
    k = torch.randn(1, 2, 16, 16, generator=g, dtype=torch.float64)
    v = torch.randn(1, 2, 16, 16, generator=g, dtype=torch.float64)
    got = BO.mixed_readout(q, k, v, frames, ws)
    want, s = 0.0, 0
    for n, w in zip(frames, ws):
        kk, vv = k[..., s: s + n, :].expand(2, -1, -1, -1), v[..., s: s + n, :].expand(2, -1, -1, -1)
        want = want + w * F.scaled_dot_product_attention(q, kk, vv)
        s += n
    assert float((got - want).abs().max()) < 1e-12
    # not a joint softmax over the union of the keys
    joint = F.scaled_dot_product_attention(q, k.expand(2, -1, -1, -1), v.expand(2, -1, -1, -1))
    assert float((got - joint).abs().max()) > 1e-3
