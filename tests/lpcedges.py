"""Inputs that reach the rarely taken branches of the encoder's LPC stage (the quantiser's edges, the precision cap, the skipped
orders, Levinson's early stop and the residual-width flags), shared by test_oracle_lpc_edges.py and test_gpu_lpc_edges.py.

Two kinds:
  * constructed autocorrelation rows, fed straight to the LPC analysis (fo_lpc_candidates in the oracle, k_lpc through
    flac_b200.debug_lpc); every branch of the quantiser can be reached this way;
  * PCM for whole encodes: noise integrated k times at 20-24 bits reaches negative shifts, coefficients clipped to qmin / qmax,
    residuals wider than 32 bits before the shift and the checked (limit) residual; a full-scale burst where the window gives
    (almost) no weight makes a checked residual leave int32 and, in partitions of 8 samples, wraps the reference's 32-bit
    partition sums."""
import numpy as np
from scipy.special import gammaln

import signals

# ---------------------------------------------------------------- constructed autocorrelations

LAGS = 33  # autocorrelation entries 0 .. 32


def ar_autoc(a, k, scale=1e12):
    """Autocorrelation (lags 0..32, autoc[0] == scale) of the impulse response h[n] = C(n+k-1, k-1) a^n of (1 - a z^-1)^-k,
    taken in closed form over its first 2^15 samples (a finite sequence, so the row is a true autocorrelation). With a close to
    1 and k large its predictor is about the binomial expansion of (1 - a z^-1)^k: coefficients up to about C(k, k/2), which
    need negative shifts at every precision."""
    n = np.arange(1 << 15, dtype=np.float64)
    logh = gammaln(n + k) - gammaln(k) - gammaln(n + 1) + n * np.log(a)
    h = np.exp(logh - logh.max())
    r = np.array([np.dot(h[:h.size - l], h[l:]) for l in range(LAGS)])
    return r * (scale / r[0])


def constructed_rows():
    """(name, autoc[0..32]) rows, each reaching some edge of the LPC stage."""
    rows = []
    for a in (0.9, 0.99, 0.999):
        for k in (1, 2, 4, 8, 12, 16, 20, 24, 28, 32):
            rows.append((f"ar a={a} k={k}", ar_autoc(a, k)))
    delta = np.zeros(LAGS)
    delta[0] = 1e9
    rows.append(("delta", delta))  # every coefficient 0: cmax == 0 at every order
    for eps in (1e-3, 1e-5, 1e-7):
        d = delta.copy()
        d[1:] = eps * 1e9 * np.cos(np.arange(1, LAGS))
        rows.append((f"near-delta {eps}", d))  # tiny coefficients: the shift clamped at 15
    rows.append(("zero", np.zeros(LAGS)))  # autoc[0] == 0: no candidate
    rows.append(("constant", np.full(LAGS, 4096.0)))  # exactly singular: error 0.0 at order 1
    rows.append(("alternating", 4096.0 * (-1.0) ** np.arange(LAGS)))
    # cos(pi l / 3): reflection coefficient exactly 1.0 at order 2, so the error reaches 0.0 at a middle order
    cos3 = np.array([1.0, 0.5, -0.5, -1.0, -0.5, 0.5] * 6)[:LAGS]
    rows.append(("cos pi/3", 2.0 ** 20 * cos3))
    rows.append(("cos pi/3 + ar", 2.0 ** 20 * cos3 + ar_autoc(0.5, 1, 2.0 ** 18)))
    # a coefficient whose scaled value is exactly .5 away from an integer: autoc [4, 1] gives 0.25 + 2^-20
    half = np.zeros(LAGS)
    half[0], half[1] = 4.0, 1.0 + 2.0 ** -18
    rows.append(("half", half))
    # a negative autoc[0] (a punch-out window whose root is smaller than its partial) with |autoc[1]| far above it: the error
    # turns positive at order 1 and the coefficient is -autoc[1] / autoc[0], here 2^21 and 2^25 -- shifts below -16
    for e in (21, 25):
        steep = np.zeros(LAGS)
        steep[0], steep[1], steep[2] = -1.0, 2.0 ** e, 3.0
        rows.append((f"steep 2^{e}", steep))
    # order-1 coefficient -(2^m - 1) (a negative autoc[0] again): at precision m + 1 it is quantised at shift 0 to 2^m - 1, and
    # at subframe bps 32 - m the prediction before the shift then fits 32 bits while the residual does not (limit without a
    # wide prediction); at higher precisions the shift is positive and the coefficient scales up towards qmax
    for m in range(4, 15):
        lim = np.zeros(LAGS)
        lim[0], lim[1] = -1.0, float((1 << m) - 1)
        rows.append((f"limit only 2^{m}-1", lim))
    assert all(np.all(np.isfinite(r)) for _, r in rows)
    return rows


# punch-out pairs (kind 1): autoc = root - partial for l < max_order, entry max_order the partial's. A root smaller than its
# partial gives a negative autoc[0]; a root that equals the partial gives 0.
def punchout_pairs():
    base = ar_autoc(0.99, 8)
    return [("root > partial", base * 2.0, base * 0.75), ("root < partial", base * 0.5, base),
            ("root == partial", base, base.copy()), ("wide root", ar_autoc(0.999, 24) * 4.0, ar_autoc(0.9, 2))]


def effective_autoc(kind, row, root, max_order, wasted, unshifted):
    """The autocorrelation k_lpc analyses for one window (as apply_apodization_ leaves it, stream_encoder.c:4339-4371),
    scaled by 2^-2w when the rows are of the signal before its wasted bits were shifted out."""
    sc = 2.0 ** (-2 * wasted) if unshifted else 1.0
    out = np.zeros(max_order + 1)
    if kind == 0:
        out[:] = row[:max_order + 1] * sc
    else:
        out[:max_order] = root[:max_order] * sc - row[:max_order] * sc
        out[max_order] = row[max_order] * sc
    return out


# ---------------------------------------------------------------- PCM

def integrated_noise(n, bps, k, seed, bs=4096):
    """White noise integrated k times, every block of bs scaled to full scale on its own (so each block is a steep, smooth
    curve whose best predictor is about (1 - z^-1)^k)."""
    rng = np.random.default_rng(seed)
    hi = (1 << (bps - 1)) - 1
    out = np.empty(n, dtype=np.int64)
    for s in range(0, n, bs):
        m = min(bs, n - s)
        v = rng.standard_normal(m + 64)
        for _ in range(k):
            v = np.cumsum(v)
            v -= np.linspace(v[0], v[-1], v.size)  # keep the block from drifting to one side
        v = v[64:]
        v = v / max(np.abs(v).max(), 1e-300) * hi
        out[s:s + m] = np.clip(np.round(v), -hi - 1, hi)
    return out


def integrated(n, ch, bps, k, seed, bs=4096, opposed=False):
    """Integrated noise on every channel; opposed: odd channels are the even ones negated (plus one LSB of noise), so that at
    24 bits left - right needs 25 bits."""
    x = np.empty((n, ch), dtype=np.int64)
    rng = np.random.default_rng(seed + 7)
    hi, lo = (1 << (bps - 1)) - 1, -(1 << (bps - 1))
    for c in range(ch):
        if opposed and c % 2 == 1:
            x[:, c] = np.clip(-x[:, c - 1] + rng.integers(-1, 2, size=n), lo, hi)
        else:
            x[:, c] = integrated_noise(n, bps, k + c % 3, seed + c, bs)
    return np.ascontiguousarray(x.astype(np.int32))


def with_bursts(x, bps, bs, where, width=6, seed=0):
    """A full-scale alternating burst of `width` samples in every full block of x: where='end' puts it at the block's last
    samples (weight ~0 under tukey(0.5)), where='middle' inside the zeroed middle third of punchout_tukey(3)."""
    x = x.copy()
    hi, lo = (1 << (bps - 1)) - 1, -(1 << (bps - 1))
    rng = np.random.default_rng(seed)
    for s in range(0, x.shape[0] - bs + 1, bs):
        at = s + bs - width if where == "end" else s + bs // 2 - width // 2 + int(rng.integers(-bs // 8, bs // 8))
        burst = np.where(np.arange(width) % 2 == 0, hi, lo)
        x[at:at + width, :] = burst[:, None] if x.shape[1] == 1 else np.stack([burst if c % 2 == 0 else -burst - 1
                                                                              for c in range(x.shape[1])], axis=1)
    return x


# (name, channels, bps, level, blocksize, config overrides, x): every stream ends in a short last block. The oracle's counters
# (test_oracle_lpc_edges.py) show which edge each input reaches.
EXHAUSTIVE_32 = dict(max_lpc_order=32, do_exhaustive_model_search=1, do_qlp_coeff_prec_search=1)


def pcm_cases():
    cases = []

    def add(name, x, bps, level, bs, **cfg):
        cases.append((name, x.shape[1], bps, level, bs, cfg, x))

    # partitions of 8 samples at 24 bits: the reference sums them in 32 bits, and the burst's residuals wrap them
    add("wrap 24-bit bs 512", with_bursts(integrated(512 * 6 + 77, 1, 24, 8, seed=2, bs=512), 24, 512, "end", width=48), 24, 8, 512,
        **EXHAUSTIVE_32)
    # a checked (limit) residual that leaves int32 on the burst, the tukey window giving the burst almost no weight
    add("overflow 24-bit", with_bursts(integrated(4096 * 2 + 301, 1, 24, 8, seed=3), 24, 4096, "end", width=32), 24, 8, 4096, **EXHAUSTIVE_32)
    # the burst inside the zeroed middle of punchout_tukey(3)
    add("punch-out burst 24-bit", with_bursts(integrated(4096 * 2 + 45, 1, 24, 8, seed=4), 24, 4096, "middle", width=32), 24, 8, 4096,
        apodization="tukey(5e-1);partial_tukey(2);punchout_tukey(3)", max_lpc_order=32, do_exhaustive_model_search=1)
    # left ~ -right at 24 bits: a 25-bit side channel
    add("opposed stereo 24-bit", integrated(4096 * 2 + 1001, 2, 24, 6, seed=5, opposed=True), 24, 8, 4096, do_qlp_coeff_prec_search=1)
    add("opposed stereo 24-bit -e", with_bursts(integrated(4096 * 2 + 13, 2, 24, 9, seed=6, opposed=True), 24, 4096, "end", width=24), 24, 8,
        4096, **EXHAUSTIVE_32)
    # 17 bits (and an 18-bit side channel): the precision cap
    add("17-bit stereo", integrated(4096 * 2 + 333, 2, 17, 5, seed=7, opposed=True), 17, 8, 4096, **EXHAUSTIVE_32)
    add("16-bit mono", integrated(4096 * 2 + 5, 1, 16, 6, seed=8), 16, 8, 4096, qlp_coeff_precision=15, max_lpc_order=32,
        do_exhaustive_model_search=1)
    # 24-bit music: the chosen LPC subframes need the 64-bit residual (prediction before the shift wider than 32 bits), so the
    # emit runs its wide residual on every path, k_emit3 for one and two channels included
    add("music 24-bit mono", signals.music_like(4096 * 2 + 211, 1, 24, 44100, seed=11), 24, 8, 4096)
    add("music 24-bit stereo", signals.music_like(4096 * 2 + 29, 2, 24, 44100, seed=12), 24, 8, 4096)
    # five and seven channels: k_emit3<PAIR> + k_join
    add("5ch 24-bit", with_bursts(integrated(4096 * 2 + 19, 5, 24, 7, seed=9), 24, 4096, "end", width=32), 24, 8, 4096,
        do_qlp_coeff_prec_search=1, max_lpc_order=32)
    add("7ch 22-bit", integrated(4096 * 2 + 97, 7, 22, 8, seed=10), 22, 5, 4096, do_qlp_coeff_prec_search=1)
    return cases


def ref_opts(cfg):
    """reflib.RefEncOpts keywords for the oracle configuration overrides above."""
    names = {"max_lpc_order": "max_lpc_order", "do_exhaustive_model_search": "exhaustive", "do_qlp_coeff_prec_search": "prec_search",
             "qlp_coeff_precision": "qlp_precision", "apodization": "apodization"}
    return {names[k]: v for k, v in cfg.items()}
