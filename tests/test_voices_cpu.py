"""Host side of a voice per text (sopro_b200/voices.py): references mapped to prefill slots by identity, and every
refusal of synthesize_batch's `ref` raised before any device work, leaving the global generator untouched."""
import dataclasses

import pytest
import torch

from sopro_b200 import voices
from sopro_b200.prefill import PreparedReference

GEOM = dict(layers=3, heads=2, head_dim=192, sv_dim=192)


def _voice(Tr=5, layers=3, heads=2, dh=192, sv=192, batch_dim=True):
    shape = (1, heads, Tr, dh) if batch_dim else (heads, Tr, dh)
    caches = [{"k": torch.zeros(shape), "v": torch.zeros(shape), "key_padding_mask": None} for _ in range(layers)]
    return PreparedReference(ref_tokens_btq=torch.zeros((1, Tr, 32), dtype=torch.long), sv_ref=torch.zeros((1, sv)),
                             ref_seq=torch.zeros((1, Tr, heads * dh)), ref_kv_caches=caches)


def test_one_reference_is_one_slot_for_every_text():
    r = _voice()
    slots, of = voices.check_voices(r, 4, **GEOM)
    assert len(slots) == 1 and slots[0] is r and of == [0, 0, 0, 0]


def test_sequence_maps_to_slots_by_identity_in_first_use_order():
    a, b, c = _voice(1), _voice(37), _voice(300)
    slots, of = voices.check_voices([b, a, b, c, a, a], 6, **GEOM)
    assert [id(s) for s in slots] == [id(b), id(a), id(c)]
    assert of == [0, 1, 0, 2, 1, 1]
    # equal content, distinct objects: distinct slots (no content hashing)
    twin = dataclasses.replace(a)
    slots, of = voices.voice_slots([a, twin], 2)
    assert len(slots) == 2 and of == [0, 1]
    slots, of = voices.voice_slots((a, a, a), 3)  # a tuple works as well as a list
    assert len(slots) == 1 and of == [0, 0, 0]


def test_repeated_object_gives_one_slot():
    r = _voice(150)
    for n in (1, 2, 64):
        slots, of = voices.check_voices([r] * n, n, **GEOM)
        assert len(slots) == 1 and slots[0] is r and of == [0] * n


def test_check_voice_returns_the_reference_frames():
    assert voices.check_voice(_voice(1), **GEOM) == 1
    assert voices.check_voice(_voice(4096), **GEOM) == 4096
    assert voices.check_voice(_voice(38, batch_dim=False), **GEOM) == 38


def _refusals():
    good = _voice()
    padded = _voice()
    padded.ref_kv_caches[1]["key_padding_mask"] = torch.zeros((1, 5), dtype=torch.bool)
    ragged = _voice()
    ragged.ref_kv_caches[2] = {"k": torch.zeros((1, 2, 6, 192)), "v": torch.zeros((1, 2, 6, 192)), "key_padding_mask": None}
    kv_mismatch = _voice()
    kv_mismatch.ref_kv_caches[0]["v"] = torch.zeros((1, 2, 4, 192))
    two_rows = _voice()
    two_rows.ref_kv_caches[0]["k"] = torch.zeros((2, 2, 5, 192))
    two_rows.ref_kv_caches[0]["v"] = torch.zeros((2, 2, 5, 192))
    return [
        ("length short", [good], 2, ValueError),
        ("length long", [good, good, good], 2, ValueError),
        ("empty", [], 1, ValueError),
        ("element", [good, "voice.wav"], 2, TypeError),
        ("element none", [None, good], 2, TypeError),
        ("not a sequence", 42, 1, TypeError),
        ("a string", "ab", 2, TypeError),
        ("layers", [good, _voice(layers=2)], 2, ValueError),
        ("heads", [good, _voice(heads=4, dh=96)], 2, ValueError),
        ("head dim", [_voice(dh=96), good], 2, ValueError),
        ("sv_dim", [good, _voice(sv=128)], 2, ValueError),
        ("Tr 0", [good, _voice(Tr=0)], 2, ValueError),
        ("Tr 4097", [_voice(Tr=4097), good], 2, ValueError),
        ("Tr differs by layer", [good, ragged], 2, ValueError),
        ("K and V differ", [kv_mismatch, good], 2, ValueError),
        ("batched K", [two_rows, good], 2, ValueError),
        ("key padding mask", [good, padded], 2, NotImplementedError),
    ]


@pytest.mark.parametrize("case", range(len(_refusals())), ids=[c[0] for c in _refusals()])
def test_refusals_leave_the_global_generator_untouched(case):
    _name, ref, n, exc = _refusals()[case]
    torch.manual_seed(1234)
    before = torch.get_rng_state()
    with pytest.raises(exc):
        voices.check_voices(ref, n, **GEOM)
    assert torch.equal(torch.get_rng_state(), before)


def test_one_reference_keeps_the_prefills_own_refusals():
    """A single PreparedReference is not re-checked here: the prefill refuses it as it always has (SoproError)."""
    slots, of = voices.check_voices(_voice(Tr=4097), 2, **GEOM)
    assert len(slots) == 1 and of == [0, 0]


def test_data_parallel_slices_a_voice_per_text_with_the_texts():
    from sopro_b200.dp import DataParallelTTS

    class Rec:
        def synthesize_batch(self, texts, *, ref, seeds=None, **kw):
            self.args = (list(texts), ref, seeds)
            return ["w"] * len(texts)

    dp = DataParallelTTS.__new__(DataParallelTTS)
    dp.group, dp.world, dp.rank, dp.tts = None, 2, 1, Rec()
    refs = [_voice() for _ in range(5)]
    texts = [str(i) for i in range(5)]
    wavs, (lo, hi) = dp.synthesize_batch(texts, ref=refs, seeds=list(range(5)))
    assert (lo, hi) == (2, 5) and len(wavs) == 3
    t, r, s = dp.tts.args
    assert t == texts[2:] and s == [2, 3, 4] and len(r) == 3 and all(x is y for x, y in zip(r, refs[2:]))
    one = refs[0]
    dp.synthesize_batch(texts, ref=one)
    assert dp.tts.args[1] is one
    with pytest.raises(ValueError):
        dp.synthesize_batch(texts, ref=refs[:4])
