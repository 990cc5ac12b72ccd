"""Oracle: analyze_track's tempo, energy and key.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Restates the three librosa calls of ``tasks/analysis.py:344-365`` (analyze_track) at librosa 0.11.0
(requirements/common.txt), which is not a dependency of this project, from that release's source semantics:

    tempo, _ = librosa.beat.beat_track(y=audio, sr=sr)
    average_energy = np.mean(librosa.feature.rms(y=audio))
    chroma = librosa.feature.chroma_stft(y=audio, sr=sr)       # key / scale from its mean (key_scale below)

All three frame with n_fft 2048, hop 512, a periodic Hann and center=True with pad_mode='constant' (zero padding,
librosa >= 0.10's default), so a track of n samples has T = 1 + n // 512 frames.  What each function restates:

  stft_power          core/spectrum.py stft + _spectrogram(power=2): float32 frames x float64 window, float64 rFFT
                      stored as complex64, |.|**2 in float32.
  onset_envelope      onset/onset_strength -> onset_strength_multi(lag=1, max_size=1, detrend=False, center=True,
                      feature=melspectrogram(fmax=sr/2), aggregate=np.median): power_to_db(ref=1, amin=1e-10,
                      top_db=80) clipped against the whole track's maximum, S[:, 1:] - S[:, :-1] clamped at 0, the
                      median over the 128 mels (util.sync over one slice), left pad lag + n_fft // (2 hop) = 3 zeros,
                      trim to T.  The envelope is float32, as librosa's is for float32 audio.
  tempogram_mean      feature/rhythm.py tempogram(win_length=time_to_frames(8.0), center=True, window='hann',
                      norm=np.inf): np.pad(mode='linear_ramp', end_values=0) by win // 2, util.frame(hop 1), first T
                      frames, x periodic Hann (float64), core/audio.py autocorrelate (lags 0 .. win - 1; computed
                      here as direct float64 sums instead of an FFT), util.normalize(norm=inf) with all-zero frames
                      left 0; then tempo()'s aggregate=np.mean over frames.
  tempo_from_tempogram  feature/rhythm.py tempo(start_bpm=120, std_bpm=1, max_tempo=320, prior=None):
                      tempo_frequencies (bpm[0] = inf), the log-normal prior, -inf below argmax(bpm < 320),
                      argmax(log1p(1e6 tg) + logprior).  beat/beat_track returns 0.0 when the envelope is all zero.
  rms                 feature/spectral.py rms(frame_length=2048, hop_length=512, center=True, pad_mode='constant'):
                      sqrt(mean(x**2)) per zero-padded frame (here in float64, cast to float32).
  piptrack_peaks      core/pitch.py piptrack(fmin=150, fmax=min(4000, sr/2), threshold=0.1, ref=np.max) on S:
                      shift = _parabolic_interpolation(S) (the 0.11 numba stencil: a = x[k+1] + x[k-1] - 2 x[k],
                      b = (x[k+1] - x[k-1]) / 2, shift = 0 when |b| >= |a| else -b / a; 0 at both ends), avg =
                      np.gradient(S), mag = S + 0.5 avg shift, pitch = (k + shift) sr / n_fft stored as float32, at
                      the bins where fmin <= rfftfreq < fmax and util.localmax(S * (S > 0.1 max_k S)) holds
                      (x[k] > x[k-1] and x[k] >= x[k+1], edge-padded).  float32 throughout, as librosa's.
  tuning_from_peaks   core/pitch.py estimate_tuning(resolution=0.01, bins_per_octave=12): keep the peaks with
                      mag >= np.median(all peak mags of the track) (float32, the mean of the two middle values),
                      then pitch_tuning: residual = (12 log2(f / 27.5)) mod 1, minus 1 where >= 0.5 (here in float64),
                      np.histogram against np.linspace(-0.5, 0.5, 101) (left-closed bins, the last one closed),
                      tuning = the left edge of the first fullest bin; 0.0 without peaks.
  chroma_filterbank   filters.py chroma(n_chroma=12, tuning, ctroct=5.0, octwidth=2, norm=2, base_c=True,
                      dtype=float32).
  chroma              feature/spectral.py chroma_stft: chromafb @ S (here in float64), util.normalize(norm=inf) per
                      frame with all-zero frames left 0.
  key_scale           tasks/analysis.py:349-365 as written.

Every discrete decision comes with a margin (``track_features``): the tempo argmax's relative gap, the tuning
histogram's count gap against the peaks that a 1e-4 relative perturbation of S could move (``tuning_fragile``), and
the gap between the best and the runner-up key correlation (``key_margin``: the 24 are 12 distinct values).

PARITY: pinned against this restatement's known answers (tests/test_track_features_host.py) and against goldens made
by the reference's own analyze_track (tests/golden/make_track_features_golden.py), NOT against librosa.
"""
from __future__ import annotations

import numpy as np

from . import mel as omel

N_FFT = 2048
HOP = 512
N_MELS = 128
TOP_DB = 80.0
LAG = 1
AC_SIZE = 8.0
START_BPM = 120.0
MAX_TEMPO = 320.0
PIP_FMIN = 150.0
PIP_FMAX = 4000.0
PIP_THRESHOLD = 0.1
N_HIST = 100
PERTURB = 1e-4
KEYS = ['C', 'C#', 'D', 'D#', 'E', 'F', 'F#', 'G', 'G#', 'A', 'A#', 'B']
MAJOR = np.array([1, 0, 1, 0, 1, 1, 0, 1, 0, 1, 0, 1])
MINOR = np.array([1, 0, 1, 1, 0, 1, 0, 1, 1, 0, 1, 0])


def n_frames(n):
    return 1 + int(n) // HOP


def tempogram_win(sr):
    """time_to_frames(8.0, sr, 512): floor(int(8 sr) / 512)"""
    return int(int(AC_SIZE * sr) // HOP)


def _frames(y):
    """float32 frames [T, 2048] of the zero-padded (center=True, pad_mode='constant') signal"""
    y = np.asarray(y, dtype=np.float32)
    yp = np.pad(y, N_FFT // 2)
    T = n_frames(len(y))
    return np.lib.stride_tricks.as_strided(yp, (T, N_FFT), (HOP * 4, 4), writeable=False)


def stft_power(y, chunk=2048):
    """|STFT|^2 f32[1025, T]"""
    fr = _frames(y)
    win = omel.hann_periodic(N_FFT)
    out = np.empty((N_FFT // 2 + 1, fr.shape[0]), np.float32)
    for t0 in range(0, fr.shape[0], chunk):
        spec = np.fft.rfft(win[None, :] * fr[t0:t0 + chunk], axis=1).astype(np.complex64)
        out[:, t0:t0 + chunk] = (np.abs(spec) ** 2).T
    return out


def rms(y):
    """f32[1, T]"""
    fr = _frames(y).astype(np.float64)
    return np.sqrt(np.mean(fr * fr, axis=1)).astype(np.float32)[None, :]


def mel_db(S, sr):
    """power_to_db(melspectrogram) in float64 before the top_db clip: f64[128, T]"""
    fb = omel.mel_filterbank(sr, N_FFT, N_MELS, 0.0, sr / 2.0).astype(np.float64)
    return 10.0 * np.log10(np.maximum(1e-10, fb @ S.astype(np.float64)))


def onset_envelope(S, sr):
    """onset_strength(y, sr, aggregate=np.median): f32[T]"""
    db = mel_db(S, sr)
    T = db.shape[1]
    db = np.maximum(db, db.max() - TOP_DB)
    diff = np.maximum(0.0, db[:, LAG:] - db[:, :-LAG])
    env = np.zeros(T, np.float64)
    pad = LAG + N_FFT // (2 * HOP)
    if T > LAG:
        med = np.median(diff, axis=0)
        env[pad:] = med[:max(0, T - pad)]
    return env.astype(np.float32)


def tempogram_frames(env, sr):
    """The windowed, autocorrelated, inf-normalised frames: f64[T, win]"""
    win = tempogram_win(sr)
    env = np.asarray(env, np.float32)
    T = len(env)
    padded = np.pad(env, win // 2, mode="linear_ramp", end_values=0)
    fr = np.lib.stride_tricks.sliding_window_view(padded, win)[:T].astype(np.float64)
    fr = fr * omel.hann_periodic(win)[None, :]
    ac = np.empty((T, win), np.float64)
    for k in range(win):
        ac[:, k] = np.einsum("tj,tj->t", fr[:, :win - k], fr[:, k:])
    length = np.max(np.abs(ac), axis=1, keepdims=True)
    length[length < np.finfo(np.float64).tiny] = 1.0
    return ac / length


def tempogram_mean(env, sr):
    return np.mean(tempogram_frames(env, sr), axis=0)


def bpm_table(sr):
    win = tempogram_win(sr)
    bpm = np.zeros(win, np.float64)
    bpm[0] = np.inf
    bpm[1:] = 60.0 * sr / (HOP * np.arange(1.0, win))
    return bpm


def tempo_scores(tg, sr):
    bpm = bpm_table(sr)
    with np.errstate(divide="ignore", invalid="ignore"):
        logprior = -0.5 * ((np.log2(bpm) - np.log2(START_BPM)) / 1.0) ** 2
    logprior[:int(np.argmax(bpm < MAX_TEMPO))] = -np.inf
    return np.log1p(1e6 * np.asarray(tg, np.float64)) + logprior


def tempo_from_tempogram(tg, sr):
    """(tempo, argmax, relative margin of the best score over the runner-up)"""
    score = tempo_scores(tg, sr)
    best = int(np.argmax(score))
    finite = np.sort(score[np.isfinite(score)])
    margin = (finite[-1] - finite[-2]) / max(abs(finite[-1]), 1e-300) if len(finite) > 1 else np.inf
    return float(bpm_table(sr)[best]), best, float(margin)


def pip_bins(sr):
    """[kmin, kmax): the bins with fmin <= rfftfreq < fmax"""
    f = np.fft.rfftfreq(N_FFT, 1.0 / sr)
    m = np.flatnonzero((PIP_FMIN <= f) & (f < min(PIP_FMAX, float(sr) / 2)))
    return int(m[0]), int(m[-1]) + 1


def _parabolic_shift(S):
    """librosa 0.11 _parabolic_interpolation along axis 0, float32"""
    x = S.astype(np.float32)
    xp, x0, xm = x[2:], x[1:-1], x[:-2]
    a = (xp + xm) - np.float32(2) * x0
    b = (xp - xm) / np.float32(2)
    shift = np.zeros_like(x)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(np.abs(b) >= np.abs(a), np.float32(0), -b / a)
    shift[1:-1] = s
    return shift


def _localmax(x):
    xp = np.pad(x, ((1, 1), (0, 0)), mode="edge")
    return (x > xp[:-2]) & (x >= xp[2:])


def piptrack_peaks(S, sr):
    """Peaks of piptrack: dict of frame i64, bin i64, pitch f32, mag f32 (frame-major, ascending bin), plus what the
    fragility count needs"""
    S = np.abs(S.astype(np.float32))
    kmin, kmax = pip_bins(sr)
    ref = np.float32(PIP_THRESHOLD) * S.max(axis=0, keepdims=True)
    lm = _localmax(S * (S > ref))
    mask = np.zeros_like(lm)
    mask[kmin:kmax] = True
    shift = _parabolic_shift(S)
    avg = np.gradient(S, axis=0)
    tt, kk = np.nonzero((lm & mask).T)
    pitch = ((kk + shift[kk, tt].astype(np.float64)) * float(sr) / N_FFT).astype(np.float32)
    mag = (S[kk, tt] + (np.float32(0.5) * avg[kk, tt]) * shift[kk, tt]).astype(np.float32)
    return {"frame": tt.astype(np.int64), "bin": kk.astype(np.int64), "pitch": pitch, "mag": mag,
            "shift": shift[kk, tt], "S": S, "ref": ref[0], "kmin": kmin, "kmax": kmax}


def hist_edges():
    return np.linspace(-0.5, 0.5, N_HIST + 1)


def residuals(pitch):
    r = np.mod(12.0 * np.log2(np.asarray(pitch, np.float64) / 27.5), 1.0)
    r[r >= 0.5] -= 1.0
    return r


def median_f32(v):
    """np.median of float32 values: the middle one, or the float32 mean of the two middle ones"""
    v = np.sort(np.asarray(v, np.float32))
    n = len(v)
    if n == 0:
        return np.float32(0.0)
    if n % 2:
        return v[n // 2]
    return np.float32((v[n // 2 - 1] + v[n // 2]) / np.float32(2))


def tuning_from_peaks(peaks):
    """(tuning, threshold, residuals of the kept peaks, counts i64[100], kept mask)"""
    mag, pitch = peaks["mag"], peaks["pitch"]
    if len(mag) == 0:
        return 0.0, np.float32(0.0), np.zeros(0), np.zeros(N_HIST, np.int64), np.zeros(0, bool)
    thr = median_f32(mag)
    keep = (mag >= thr) & (pitch > 0)
    res = residuals(pitch[keep])
    counts, edges = np.histogram(res, hist_edges())
    return float(edges[int(np.argmax(counts))]), thr, res, counts, keep


def tuning_fragile(peaks, thr, counts, sr, eps=PERTURB):
    """How far the histogram's count gap could close under a relative perturbation eps of S (first order; the frame
    maximum, and with it the threshold, moves too): the tuning decision stands when the gap exceeds it.

    Peaks can appear or vanish (localmax / threshold flips, n_lm of them), cross the median (which itself moves by the
    perturbation and by n_lm ranks), and cross a histogram edge (the residual moves with the interpolated pitch).  The
    top bin keeps at least its surely-included, edge-safe peaks, and at least half of all peaks minus those that could
    be counted elsewhere; any other bin gains at most its possibly-included peaks and the edge crossers next to it."""
    S, ref = peaks["S"].astype(np.float64), peaks["ref"].astype(np.float64)
    kmin, kmax = peaks["kmin"], peaks["kmax"]
    x = S[kmin - 1:kmax + 1]
    up, dn = 1.0 + 2 * eps, 1.0 - 2 * eps
    c, l, r = x[1:-1], x[:-2], x[2:]
    # optimistic: centre up, neighbours and threshold down; pessimistic: the reverse
    pk_hi = (c * up > ref * dn) & (c * up > l * dn * (l * dn > ref * dn)) & (c * up >= r * dn * (r * dn > ref * dn))
    pk_lo = (c * dn > ref * up) & (c * dn > l * up * (l * up > ref * up)) & (c * dn >= r * up * (r * up > ref * up))
    n_lm = int(np.count_nonzero(pk_hi != pk_lo))
    mag = peaks["mag"].astype(np.float64)
    N = len(mag)
    srt = np.sort(mag)
    d = 2 * eps
    thr_lo = srt[max(0, (N - 1) // 2 - n_lm)] * (1 - d)
    thr_hi = srt[min(N - 1, N // 2 + n_lm)] * (1 + d)
    sure_in = mag * (1 - d) >= thr_hi
    poss_in = mag * (1 + d) >= thr_lo
    # histogram bin: the residual moves with the interpolated pitch; bound d(shift) to first order
    kk, tt = peaks["bin"], peaks["frame"]
    xp, x0, xm = S[kk + 1, tt], S[kk, tt], S[kk - 1, tt]
    a = xp + xm - 2 * x0
    sh = peaks["shift"].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        dsh = eps * ((np.abs(xp) + np.abs(xm)) / 2 + np.abs(sh) * (np.abs(xp) + np.abs(xm) + 2 * np.abs(x0))) / np.abs(a)
        dsh = np.where(np.isfinite(dsh), dsh, 1.0)
    dres = 12.0 / np.log(2.0) * dsh / (kk + sh) + 4e-5     # + float32 rounding of librosa's log2 / mod
    res = residuals(peaks["pitch"])
    edges = hist_edges()
    b = np.clip(np.searchsorted(edges, res, side="right") - 1, 0, N_HIST - 1)
    dl, dr = res - edges[b], edges[b + 1] - res
    frag = np.minimum(dl, dr) <= dres
    alt = np.where(dl <= dr, (b - 1) % N_HIST, (b + 1) % N_HIST)
    top = int(np.argmax(counts))
    safe_top = (b == top) & ~frag
    lower_top = max(int(np.count_nonzero(sure_in & safe_top)),
                    -(-(N - n_lm) // 2) - int(np.count_nonzero(poss_in & ~safe_top)))
    upper = np.zeros(N_HIST, np.int64)
    np.add.at(upper, b[poss_in], 1)
    np.add.at(upper, alt[poss_in & frag], 1)
    upper += n_lm
    upper[top] = -1
    runner = np.sort(counts)[-2]
    return int(counts[top] - lower_top) + int(upper.max() - runner)


def chroma_filterbank(sr, tuning, n_chroma=12):
    """filters.chroma(sr, 2048, tuning=tuning): f32[12, 1025]"""
    frequencies = np.linspace(0, sr, N_FFT, endpoint=False)[1:]
    a440 = 440.0 * 2.0 ** (tuning / n_chroma)
    frqbins = n_chroma * np.log2(frequencies / (a440 / 16))
    frqbins = np.concatenate(([frqbins[0] - 1.5 * n_chroma], frqbins))
    binwidthbins = np.concatenate((np.maximum(frqbins[1:] - frqbins[:-1], 1.0), [1]))
    D = np.subtract.outer(frqbins, np.arange(0, n_chroma, dtype="d")).T
    n_chroma2 = np.round(float(n_chroma) / 2)
    D = np.remainder(D + n_chroma2 + 10 * n_chroma, n_chroma) - n_chroma2
    wts = np.exp(-0.5 * (2 * D / np.tile(binwidthbins, (n_chroma, 1))) ** 2)
    length = np.sum(wts ** 2, axis=0, keepdims=True) ** 0.5
    length[length < np.finfo(np.float64).tiny] = 1.0
    wts = wts / length
    wts *= np.tile(np.exp(-0.5 * (((frqbins / n_chroma - 5.0) / 2) ** 2)), (n_chroma, 1))
    wts = np.roll(wts, -3 * (n_chroma // 12), axis=0)
    return np.ascontiguousarray(wts[:, :int(1 + N_FFT / 2)], dtype=np.float32)


def chroma(S, fb):
    """f64[12, T]: fb @ S normalised per frame by its max"""
    raw = fb.astype(np.float64) @ S.astype(np.float64)
    length = np.max(np.abs(raw), axis=0, keepdims=True)
    length[length < np.finfo(np.float32).tiny] = 1.0
    return raw / length


def key_correlations(chroma_mean):
    cm = np.asarray(chroma_mean, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        maj = np.array([np.corrcoef(cm, np.roll(MAJOR, i))[0, 1] for i in range(12)])
        mnr = np.array([np.corrcoef(cm, np.roll(MINOR, i))[0, 1] for i in range(12)])
    return maj, mnr


def key_scale(chroma_mean):
    """tasks/analysis.py:349-365: (key, scale, major correlations, minor correlations)"""
    maj, mnr = key_correlations(chroma_mean)
    i, j = int(np.argmax(maj)), int(np.argmax(mnr))
    if maj[i] > mnr[j]:
        return KEYS[i], "major", maj, mnr
    return KEYS[j], "minor", maj, mnr


def key_margin(maj, mnr):
    """Best minus runner-up of the distinct correlations.  Each major profile is its relative minor's profile
    (np.roll(MAJOR, i) == np.roll(MINOR, i + 9)), so the 24 correlations are 12 values twice: the best major and the
    best minor are always equal, analysis.py:360's strict `>` fails, and the reference always answers the relative
    minor of the best major key.  The margin is therefore taken over the 12 major correlations."""
    v = np.sort(maj)
    return float(v[-1] - v[-2]) if np.all(np.isfinite(v)) else 0.0


def track_features(y, sr=16000):
    """Every intermediate and decision of the three calls for one track (float32 samples)."""
    y = np.asarray(y, np.float32)
    S = stft_power(y)
    out = {"T": S.shape[1], "S": S}
    env = onset_envelope(S, sr)
    out["onset_env"] = env
    if not env.any():
        out.update(tempogram_mean=np.zeros(tempogram_win(sr)), tempo=0.0, tempo_index=0, tempo_margin=np.inf,
                   tempo_score=np.full(tempogram_win(sr), np.nan))
    else:
        tg = tempogram_mean(env, sr)
        tempo, best, margin = tempo_from_tempogram(tg, sr)
        out.update(tempogram_mean=tg, tempo=tempo, tempo_index=best, tempo_margin=margin,
                   tempo_score=tempo_scores(tg, sr))
    out["rms"] = rms(y)
    out["energy"] = float(np.mean(out["rms"]))
    peaks = piptrack_peaks(S, sr)
    tuning, thr, res, counts, keep = tuning_from_peaks(peaks)
    srt = np.sort(counts)
    fragile = tuning_fragile(peaks, thr, counts, sr) if len(peaks["mag"]) else 0
    out.update(peaks={k: peaks[k] for k in ("frame", "bin", "pitch", "mag")}, threshold=thr, residuals=res,
               histogram=counts, tuning=tuning, tuning_gap=int(srt[-1] - srt[-2]), tuning_fragile=int(fragile))
    fb = chroma_filterbank(sr, tuning)
    ch = chroma(S, fb)
    cm = np.mean(ch.astype(np.float32), axis=1)
    key, scale, maj, mnr = key_scale(cm)
    out.update(chroma_fb=fb, chroma=ch, chroma_mean=cm, key=key, scale=scale, major_corr=maj, minor_corr=mnr,
               key_margin=key_margin(maj, mnr))
    return out


# ------------------------------------------------------------------------------------------------ seeded test signals
def synth_track(kind, seconds, sr=16000, seed=0):
    """Seeded music-like float32 waveforms for tests and benchmarks.  Every kind but silence carries a sustained
    harmony, pitch classes root + {0, 4, 5, 7, 11} (only the root's major scale holds all five) tuned c cents off
    A440, c a seeded histogram-bin centre, so that tuning and key are well defined.

    'drums'    a kick / snare / hat loop at a seeded tempo, with noise
    'chord'    the harmony re-struck every half beat
    'detuned'  a dominant partial at 3520 Hz * 2^(c/1200) over a quiet harmony
    'clicks'   a click every k hops (bpm = 60 sr / (512 k)), k seeded in [12, 24], over a quiet harmony
    'silence'  zeros"""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    t = np.arange(n) / sr
    y = np.zeros(n, np.float64)
    if kind == "silence":
        return y.astype(np.float32)
    cents = float(rng.integers(-45, 45)) + 0.5
    a4 = 440.0 * 2.0 ** (cents / 1200)
    root = int(rng.integers(0, 12))
    level = {"drums": 0.12, "chord": 0.15, "detuned": 0.12, "clicks": 0.02}[kind]
    for semis, w in zip((0, 4, 5, 7, 11), (1.0, 0.8, 0.5, 0.8, 0.5)):
        f = a4 * 2.0 ** ((root + semis - 9) / 12.0)
        y += level * w * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    if kind == "clicks":
        k = int(rng.integers(12, 25))
        y[::k * HOP] += 1.0
    elif kind == "detuned":
        y += 0.4 * np.sin(2 * np.pi * 3520.0 * 2.0 ** (cents / 1200) * t)
    else:
        bpm = float(rng.uniform(80, 160))
        onsets = np.arange(0.0, seconds, 30.0 / bpm)
        for i, o in enumerate(onsets):
            s = int(o * sr)
            m = min(n - s, int(0.25 * sr))
            if m <= 0:
                continue
            env = np.exp(-np.arange(m) / (0.03 * sr))
            if kind == "drums":
                if i % 4 == 0:
                    y[s:s + m] += 0.8 * env * np.sin(2 * np.pi * 60 * np.arange(m) / sr)
                elif i % 4 == 2:
                    y[s:s + m] += 0.4 * env * rng.standard_normal(m)
                y[s:s + m] += 0.15 * env * rng.standard_normal(m) * (np.arange(m) < 0.02 * sr)
            else:
                y[s:s + m] *= 1.0 + 2.0 * env
        y += 0.01 * rng.standard_normal(n)
    return (y / max(1.0, np.abs(y).max())).astype(np.float32)
