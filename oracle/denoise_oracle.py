"""Reference-voice denoising restated in numpy float64 (sopro_b200/csrc/denoise.cu, include/sopro_b200.h): a
stationary-noise Wiener suppressor with the decision-directed a priori SNR estimate (Ephraim-Malah), over 512-sample
sqrt-Hann frames at hop 256 of a 24 kHz row."""
from __future__ import annotations

import numpy as np

N, R = 512, 256
BINS = N // 2 + 1
ALPHA = 0.98
G_MIN = 0.1  # -20 dB


def window() -> np.ndarray:
    """w[j] = sqrt(0.5 - 0.5 cos(2 pi j / N)), the periodic sqrt-Hann; w^2 at hop N/2 sums to 1."""
    j = np.arange(N, dtype=np.float64)
    return np.sqrt(0.5 - 0.5 * np.cos(2.0 * np.pi * j / N))


def n_frames(n: int) -> int:
    """M = ceil(n / R) + 1; frame m covers samples [(m - 1) R, (m + 1) R)."""
    return -(-n // R) + 1


def candidates(n: int) -> int:
    """C = floor(n / R) - 1: frames m = 1 .. C lie wholly inside the clip."""
    return n // R - 1


def n_noise(n: int) -> int:
    return max(1, candidates(n) // 10)


def analyze(x: np.ndarray) -> np.ndarray:
    """X [M][BINS] complex128 of the windowed frames (zeros outside the row)."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    n = x.size
    M = n_frames(n)
    pad = np.zeros((M + 1) * R, dtype=np.float64)
    pad[R:R + n] = x
    idx = np.arange(M)[:, None] * R + np.arange(N)[None, :]
    return np.fft.rfft(pad[idx] * window()[None, :], axis=1)


def frame_energy(P: np.ndarray) -> np.ndarray:
    """E[m] = sum over k ascending of P[m][k]."""
    E = np.zeros(P.shape[0], dtype=np.float64)
    for k in range(P.shape[1]):
        E = E + P[:, k]
    return E


def noise_frames(E: np.ndarray, n: int) -> np.ndarray:
    """The K quietest candidate frames, ascending (ties to the lower m)."""
    C = candidates(n)
    m = np.arange(1, C + 1)
    order = np.lexsort((m, E[1:C + 1]))  # by E, then by m
    return np.sort(m[order[: n_noise(n)]])


def noise_psd(P: np.ndarray, sel: np.ndarray) -> np.ndarray:
    """lambda[k] = the mean of P[m][k] over the selected frames, summed with m ascending."""
    lam = np.zeros(P.shape[1], dtype=np.float64)
    for m in sel:
        lam = lam + P[m]
    return lam / len(sel)


def gains(P: np.ndarray, lam: np.ndarray) -> np.ndarray:
    """G [M][BINS]: the decision-directed recursion over the frames; G = 1 in a bin where lambda = 0."""
    M = P.shape[0]
    G = np.ones_like(P)
    live = lam > 0
    safe = np.where(live, lam, 1.0)
    g_prev = gam_prev = None
    for m in range(M):
        gam = P[m] / safe
        post = np.maximum(gam - 1.0, 0.0)
        xi = post if m == 0 else ALPHA * g_prev * g_prev * gam_prev + (1.0 - ALPHA) * post
        g = np.maximum(xi / (1.0 + xi), G_MIN)
        G[m] = np.where(live, g, 1.0)
        g_prev, gam_prev = g, gam
    return G


def synthesize(X: np.ndarray, G: np.ndarray, n: int) -> np.ndarray:
    """Inverse real FFT of G X, windowed, overlap-added: y[i] = frame q's second half + frame q + 1's first half."""
    f = np.fft.irfft(G * X, n=N, axis=1) * window()[None, :]
    i = np.arange(n)
    q, r = i // R, i % R
    return f[q, R + r] + f[q + 1, r]


def denoise_detail(x: np.ndarray) -> dict:
    """y and how it was reached: E, the selected frames (None for a pass-through row), lambda and G."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    n = x.size
    out = {"y": x.copy(), "E": None, "sel": None, "lam": None, "G": None}
    if n < N:
        return out
    with np.errstate(invalid="ignore", over="ignore"):  # a non-finite row passes through
        X = analyze(x)
        P = X.real * X.real + X.imag * X.imag
        E = frame_energy(P)
    out["E"] = E
    if not np.isfinite(E).all():
        return out
    sel = noise_frames(E, n)
    lam = noise_psd(P, sel)
    G = gains(P, lam)
    out.update(sel=sel, lam=lam, G=G, y=synthesize(X, G, n))
    return out


def denoise(x: np.ndarray) -> np.ndarray:
    return denoise_detail(x)["y"]


def round_trip(x: np.ndarray) -> np.ndarray:
    """Analysis then synthesis with G = 1: the input again, up to rounding."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    X = analyze(x)
    return synthesize(X, np.ones(X.shape, dtype=np.float64), x.size)


# ---- the test signals of DESIGN.md §5n, all at 24 kHz

SR = 24000


def voiced(seconds: float = 6.0, gated: bool = True) -> np.ndarray:
    """A gliding 140 +- 20 Hz harmonic complex (24 harmonics, 1/k amplitudes), amplitude-modulated at 3 Hz by |sin|,
    gated to zero about half the time when `gated` (else never below 30 % amplitude), peak 0.5."""
    n = int(seconds * SR)
    t = np.arange(n) / SR
    f0 = 140.0 + 20.0 * np.sin(2 * np.pi * 0.5 * t)
    ph = 2 * np.pi * np.cumsum(f0) / SR
    s = sum(np.sin(k * ph) / k for k in range(1, 25))
    env = np.abs(np.sin(2 * np.pi * 1.5 * t))  # |sin| at 3 Hz
    if gated:
        env = np.where(np.sin(2 * np.pi * 0.4 * t + 0.3) > 0.3, env, 0.0)
    else:
        env = 0.3 + 0.7 * env
    s = s * env
    return 0.5 * s / np.abs(s).max()


def white(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).standard_normal(n)


def pink(n: int, seed: int) -> np.ndarray:
    """1/f power noise: white noise shaped by 1/sqrt(f) in the frequency domain."""
    w = np.fft.rfft(white(n, seed))
    f = np.arange(w.size, dtype=np.float64)
    f[0] = 1.0
    return np.fft.irfft(w / np.sqrt(f), n=n)


def at_snr(s: np.ndarray, noise: np.ndarray, snr_db: float) -> np.ndarray:
    """noise scaled so that the clean signal's power over the noise's is snr_db."""
    ps, pn = float(np.mean(s * s)), float(np.mean(noise * noise))
    return noise * np.sqrt(ps / (pn * 10.0 ** (snr_db / 10.0)))


def snr_db(clean: np.ndarray, y: np.ndarray) -> float:
    e = y - clean
    return 10.0 * np.log10(float(np.sum(clean * clean)) / float(np.sum(e * e)))
