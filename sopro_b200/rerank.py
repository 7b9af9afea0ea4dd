"""Best-of-N synthesis: the host side of choosing one take among N candidates of the same text.

Each text is generated N times side by side in one batch (candidate k with seed s + k), every take's NAR codes are
scored by the speaker encoder Token2SV against the reference voice's ``sv_ref`` (one launch of
``RefPrepEngine.speaker_vectors``), and only the chosen take of each text is decoded.  This module holds the argument
check, the seed mapping and the choice rule; all of it is host-only."""
from __future__ import annotations

from typing import List, Optional, Sequence

MAX_BEST_OF = 16


def check_best_of(best_of) -> int:
    """The number of candidates per text, an int in [1, 16]; ValueError otherwise (a bool is refused)."""
    if isinstance(best_of, bool) or not isinstance(best_of, int):
        raise ValueError(f"best_of must be an int in [1, {MAX_BEST_OF}], got {best_of!r}")
    if not 1 <= best_of <= MAX_BEST_OF:
        raise ValueError(f"best_of must be in [1, {MAX_BEST_OF}], got {best_of}")
    return int(best_of)


def check_rows(rows: int, limit: Optional[int]) -> None:
    """ValueError when `rows` candidate rows exceed the AR session's batch limit (None: no limit known)."""
    if limit is not None and rows > limit:
        raise ValueError(f"{rows} candidate rows exceed the batch limit of {limit}; lower best_of or the number of texts")


def candidate_seeds(seeds: Optional[Sequence[int]], best_of: int) -> Optional[List[int]]:
    """Row i*N + k of the candidate batch is candidate k of text i, with seed seeds[i] + k; None without seeds (the
    rows then draw from the global generator in that row order)."""
    if seeds is None:
        return None
    return [int(s) + k for s in seeds for k in range(int(best_of))]


def choose(Ts: Sequence[int], stopped: Sequence[bool], text_len: int, cos: Optional[Sequence[float]]) -> int:
    """The index of the take to keep among one text's candidates.

    Ts[k]: frames of candidate k before its first EOS; stopped[k]: an EOS was sampled (the take did not run out of
    frames); text_len: the text's token count; cos[k]: cosine of the take's speaker vector with the reference voice's
    (None, or ignored entries, where T = 0).

    A candidate is eligible when it stopped, has T > 0 and has T >= text_len (fewer frames than text tokens is the case
    where the word aligner finds no path: the take is certainly truncated).  The eligible candidate with the highest
    cosine wins; without one, the highest cosine among the candidates with T > 0; when every T is 0, candidate 0.
    Ties go to the lowest index."""
    n = len(Ts)
    if n < 1 or len(stopped) != n or (cos is not None and len(cos) != n):
        raise ValueError("choose needs one T, one stop flag and one cosine per candidate")
    live = [k for k in range(n) if int(Ts[k]) > 0]
    if not live:
        return 0
    eligible = [k for k in live if stopped[k] and int(Ts[k]) >= int(text_len)]
    pool = eligible or live
    best = pool[0]
    for k in pool[1:]:
        if float(cos[k]) > float(cos[best]):
            best = k
    return best
