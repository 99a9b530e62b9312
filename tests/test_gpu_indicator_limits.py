"""Indicator kernels at their limits, against the float64 restatement of `ta` (oracle/indicators_ref.py).

Price scales from ~6e-6 to ~1e5, every window bound at every tile seam, 64- and 128-window banks, and rows that are not
a dense [S][N] tensor: padded rows, odd row strides, rows off 16-byte alignment, inputs with different row strides.
"""
import ctypes
import itertools
import math

import numpy as np
import pandas as pd
import pytest

from abi_header import EINVAL, ELIMIT
from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

# kernel constants (csrc/indicators.cu, csrc/indicators2.cu)
IND_TILE, IND_MAX_WINDOW, IND_MAX_P = 2048, 1024, 64
RSI_TILE, RSI_MAX_P = 4096, 128
MACD_MAX_SPAN = 512
SMEM_LIMIT = 200 * 1024          # the host wrappers' shared-memory budget per CTA, in bytes

RTOL = 2e-6         # fp64 evaluation rounded once to fp32 vs float64 pandas
PRICE_ATOL = 1e-9   # absolute bound of price-valued outputs, as a fraction of the row's median price
UNITLESS_TOL = {    # (rtol, atol) of the unitless outputs: the bounds of tests/test_gpu_indicators.py
    "rsi": (RTOL, 1e-12), "stoch_k": (RTOL, 1e-5), "stoch_d": (RTOL, 1e-5), "williams_r": (RTOL, 1e-5),
    "bb_width": (2e-5, 1e-7), "bb_position": (2e-5, 1e-6),
}
PRICE_VALUED = {"ema", "sma", "atr", "macd_line", "macd_signal", "macd_diff", "bb_high", "bb_mid", "bb_low", "ichimoku_a",
                "ichimoku_b", "vwap", "sma_20", "sma_50", "sma_200", "ema_12", "ema_26", "macd"}


def _halo(om):
    """halo_for (indicators2.cu): bars after which om^L <= 2^-60, a multiple of 4."""
    if not om > 0:
        return 4
    return (math.ceil(60 * math.log(2) / -math.log(om)) + 3) & ~3


def _ema_halo(w):
    return _halo(1 - 2 / (w + 1))


def _wilder_halo(w):
    return _halo((w - 1) / w)


def _rsi_halo(w):
    """halo_for_alpha (indicators.cu): a multiple of 32; window 1 keeps 4 bars."""
    return 4 if w == 1 else (math.ceil(60 * math.log(2) / -math.log1p(-1 / w)) + 31) & ~31


# b200bt_atr_bank stages the true range over the longest window's warm-up halo, the tile and IND_MAX_WINDOW more bars as
# float64 in shared memory: (halo + IND_TILE + IND_MAX_WINDOW + 8) * 8 bytes <= SMEM_LIMIT holds windows up to 541
# (halo 22480 bars); window 542 (halo 22524) is refused.
ATR_MAX_WINDOW = max(w for w in range(1, IND_MAX_WINDOW + 1)
                     if (_wilder_halo(w) + IND_TILE + IND_MAX_WINDOW + 8) * 8 <= SMEM_LIMIT)
assert ATR_MAX_WINDOW == 541


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------
def _ohlcv(S, N, seed=11, trend=(), scales=None):
    """float32 [5][S][N] around 100 (0.1 % random-walk steps, high / low around open and close, lognormal volume).  Symbols
    in `trend` drift +20 % over the second 2048-bar tile; `scales[s]` multiplies symbol s's prices (in float64)."""
    rng = np.random.default_rng(seed)
    steps = rng.normal(0.0, 1e-3, (S, N))
    for s in trend:
        steps[s, IND_TILE:2 * IND_TILE] += math.log(1.2) / IND_TILE
    close = 100.0 * np.exp(np.cumsum(steps, axis=1))
    open_ = np.concatenate([close[:, :1], close[:, :-1]], axis=1)
    high = np.maximum(open_, close) * (1.0 + np.abs(rng.normal(0.0, 5e-4, (S, N))))
    low = np.minimum(open_, close) * (1.0 - np.abs(rng.normal(0.0, 5e-4, (S, N))))
    vol = rng.lognormal(5.0, 1.0, (S, N))
    prices = np.stack([open_, high, low, close])
    if scales is not None:
        prices = prices * np.asarray(scales, dtype=np.float64)[None, :, None]
    return np.concatenate([prices, vol[None]]).astype(np.float32)


def _scaled(ohlcv, k, volume_k=0):
    """Prices times 2^k, volume times 2^volume_k: exact in fp32 at these magnitudes."""
    out = ohlcv.copy()
    out[:4] *= np.float32(2.0 ** k)
    out[4] *= np.float32(2.0 ** volume_k)
    return out


def _two_scales(N, seed=11):
    """Symbol 0 at ~6e-6 (x 2^-24), symbol 1 at ~1e5 (x 2^10) with its second tile drifting 20 %."""
    d = _ohlcv(2, N, seed=seed, trend=(1,))
    d[:4, 0] *= np.float32(2.0 ** -24)
    d[:4, 1] *= np.float32(2.0 ** 10)
    return d


def _dev(torch, ohlcv):
    return [torch.from_numpy(np.ascontiguousarray(ohlcv[f])).cuda() for f in range(5)]


def _series(ohlcv, s):
    return [pd.Series(ohlcv[f, s].astype(np.float64)) for f in range(5)]


# ---------------------------------------------------------------------------------------------------------------------
# one call of an entry point (device) and its float64 restatement (one symbol); both -> {output name: array}
# ---------------------------------------------------------------------------------------------------------------------
def _gpu(entry, p, t):
    """entry point `entry` with parameters `p` on device rows t = (open, high, low, close, volume) -> numpy outputs,
    [S][P][N] for the banks, [S][N] otherwise; NaN left in place."""
    from ai_crypto_trader_b200 import indicators as ind
    from ai_crypto_trader_b200.sweep import rsi_bank
    _, h, l, c, v = t
    if entry == "ema":
        r = {"ema": ind.ema_bank(c, p, fill=False)}
    elif entry == "sma":
        r = {"sma": ind.sma_bank(c, p, fill=False)}
    elif entry == "atr":
        r = {"atr": ind.atr_bank(h, l, c, p)}
    elif entry == "rsi":
        r = {"rsi": rsi_bank(c, p, fill=False)}
    elif entry == "macd":
        r = dict(zip(("macd_line", "macd_signal", "macd_diff"), ind.macd(c, *p, fill=False)))
    elif entry == "bollinger":
        r = dict(zip(("bb_high", "bb_mid", "bb_low", "bb_width", "bb_position"), ind.bollinger(c, p, 2.0, fill=False)))
    elif entry == "stochastic":
        r = dict(zip(("stoch_k", "stoch_d"), ind.stochastic(h, l, c, *p, fill=False)))
    elif entry == "williams_r":
        r = {"williams_r": ind.williams_r(h, l, c, p, fill=False)}
    elif entry == "ichimoku":
        r = dict(zip(("ichimoku_a", "ichimoku_b"), ind.ichimoku(h, l, *p, fill=False)))
    elif entry == "vwap":
        r = {"vwap": ind.vwap(h, l, c, v, p, fill=False)}
    else:
        raise KeyError(entry)
    return {k: x.cpu().numpy() for k, x in r.items()}


def _ref(entry, p, series):
    from oracle import indicators_ref as ref
    _, h, l, c, v = series
    if entry in ("ema", "sma", "atr", "rsi"):
        f = {"ema": lambda w: ref.ema(c, w), "sma": lambda w: ref.sma(c, w), "atr": lambda w: ref.atr(h, l, c, w),
             "rsi": lambda w: ref.rsi(c, w)}[entry]
        return {entry: np.stack([f(int(w)).to_numpy() for w in p])}
    if entry == "macd":
        return dict(zip(("macd_line", "macd_signal", "macd_diff"), ref.macd(c, *p)))
    if entry == "bollinger":
        hb, mb, lb = ref.bollinger(c, p, 2.0)
        wd, pos = ref.bollinger_width_position(c, hb, mb, lb)
        return {"bb_high": hb, "bb_mid": mb, "bb_low": lb, "bb_width": wd, "bb_position": pos}
    if entry == "stochastic":
        return dict(zip(("stoch_k", "stoch_d"), ref.stochastic(h, l, c, *p)))
    if entry == "williams_r":
        return {"williams_r": ref.williams_r(h, l, c, p)}
    if entry == "ichimoku":
        return dict(zip(("ichimoku_a", "ichimoku_b"), ref.ichimoku(h, l, *p)))
    if entry == "vwap":
        return {"vwap": ref.vwap(h, l, c, v, p)}
    raise KeyError(entry)


def _tol(name, median_price):
    if name in PRICE_VALUED:
        return RTOL, PRICE_ATOL * median_price
    return UNITLESS_TOL[name]


def _cmp(got, want, what, rtol, atol):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    bad = np.flatnonzero(np.isnan(got) != np.isnan(want))
    assert bad.size == 0, (what, "NaN pattern differs at bars", bad[:8])
    m = ~np.isnan(want)
    np.testing.assert_allclose(got[m], want[m], rtol=rtol, atol=atol, err_msg=str(what))


def _check_against_ref(entry, p, ohlcv, got, label):
    for s in range(ohlcv.shape[1]):
        want = _ref(entry, p, _series(ohlcv, s))
        med = float(np.median(ohlcv[3, s]))
        for name, w in want.items():
            rtol, atol = _tol(name, med)
            _cmp(got[name][s], np.asarray(w), (label, name, "symbol", s), rtol, atol)


def _same_bits(a, b):
    """Bitwise equality, NaN payloads included."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# every per-indicator entry point, with windows from 1 to each bound
CALLS = [
    ("ema", [1, 2, 12, 26, IND_MAX_WINDOW]),
    ("sma", [1, 2, 20, 200, IND_MAX_WINDOW]),
    ("atr", [1, 2, 14, ATR_MAX_WINDOW]),
    ("rsi", [1, 2, 14, 1100, RSI_TILE]),
    ("macd", (12, 26, 9)),
    ("macd", (1, MACD_MAX_SPAN, MACD_MAX_SPAN)),
    ("bollinger", 1),
    ("bollinger", 20),
    ("bollinger", IND_MAX_WINDOW),
    ("stochastic", (14, 3)),
    ("williams_r", 14),
    ("ichimoku", (9, 26, 52)),
    ("vwap", 14),
    ("vwap", IND_MAX_WINDOW),
]


def _all_outputs(torch, ohlcv, analyzer=True):
    """{(call index, output name): numpy} over CALLS, plus {("analyzer", column): numpy} from TechnicalAnalyzer."""
    from ai_crypto_trader_b200.indicators import TechnicalAnalyzer
    from ai_crypto_trader_b200.sweep import MarketData
    t = _dev(torch, ohlcv)
    out = {}
    for i, (entry, p) in enumerate(CALLS):
        for name, x in _gpu(entry, p, t).items():
            out[(i, name)] = x
    if analyzer:
        ta = TechnicalAnalyzer(MarketData(ohlcv))
        for name, x in ta.data.items():
            out[("analyzer", name)] = x.cpu().numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. price-scale equivariance, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [-24, -12, 10])
def test_price_scale_equivariance_is_bit_exact(torch_cuda, k):
    """All arithmetic is fp64 with one rounding to fp32 at the end, and no kernel holds an absolute constant at price scale
    (rsi_value's 1e-290 guard on U + D sits ~280 decades below these prices' moves).  So prices x 2^k scale every
    price-valued output by exactly 2^k and leave RSI, %K, %D, Williams %R, bb_width and bb_position unchanged; volume x 2^k
    changes nothing at all."""
    torch = torch_cuda
    data = _ohlcv(2, 9001, trend=(1,))
    base = _all_outputs(torch, data)
    scaled = _all_outputs(torch, _scaled(data, k))
    f = np.float32(2.0 ** k)
    for key, got in scaled.items():
        want = base[key] * f if key[1] in PRICE_VALUED else base[key]
        assert _same_bits(got, want), (k, CALLS[key[0]] if key[0] != "analyzer" else "analyzer", key[1],
                                       int(np.sum(~((got == want) | (np.isnan(got) & np.isnan(want))))))
    by_volume = _all_outputs(torch, _scaled(data, 0, volume_k=k))
    for key, got in by_volume.items():
        assert _same_bits(got, base[key]), (k, "volume", key)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the float64 reference at ~6e-6 and ~1e5, tolerances relative to the price
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [-24, 10])
def test_kernels_match_the_float64_reference_at_price_scale(torch_cuda, k):
    """Every entry point and the fused analyzer at prices x 2^k; symbol 0's second tile drifts 20 % (at 2^10: 1e5 -> 1.2e5
    within one 2048-bar tile, Bollinger's m2 - m1^2 on tile-offset prefixes)."""
    torch = torch_cuda
    from oracle import indicators_ref as ref
    data = _scaled(_ohlcv(2, 12000, seed=5, trend=(0,)), k)
    got = _all_outputs(torch, data)
    for i, (entry, p) in enumerate(CALLS):
        one = {name: x for (j, name), x in got.items() if j == i}
        _check_against_ref(entry, p, data, one, (k, entry, p))
    for s in range(2):
        so, sh, sl, sc, sv = _series(data, s)
        want = ref.analyzer_columns(so, sh, sl, sc, sv)
        med = float(np.median(data[3, s]))
        for name, w in want.items():
            rtol, atol = _tol(name, med)
            _cmp(got[("analyzer", name)][s], w.to_numpy(), (k, "analyzer", name, s), rtol, atol)


# ---------------------------------------------------------------------------------------------------------------------
# 3. every window bound at every tile seam
# ---------------------------------------------------------------------------------------------------------------------
def _seam_halo(entry, p):
    """Warm-up bars the entry point reads before a tile (its kernel's halo)."""
    if entry == "ema":
        return _ema_halo(max(p))
    if entry == "atr":
        return _wilder_halo(max(p))
    if entry == "rsi":
        return _rsi_halo(max(p))
    if entry == "macd":
        return _ema_halo(max(p[0], p[1])) + _ema_halo(p[2])
    if entry == "stochastic":
        return max(p) - 1 + p[1] - 1
    if entry == "ichimoku":
        return max(p) - 1
    return (max(p) if isinstance(p, list) else p) - 1         # sma, bollinger, williams_r, vwap


BOUNDS = (
    [("ema", [w]) for w in (1, 2, IND_MAX_WINDOW)]
    + [("sma", [w]) for w in (1, 2, IND_MAX_WINDOW)]
    + [("atr", [w]) for w in (1, 2, ATR_MAX_WINDOW)]
    + [("rsi", [w]) for w in (1, 2, RSI_TILE)]
    + [("macd", (w, 26, 9)) for w in (1, 2, MACD_MAX_SPAN)]
    + [("macd", (12, w, 9)) for w in (1, 2, MACD_MAX_SPAN)]
    + [("macd", (12, 26, w)) for w in (1, 2, MACD_MAX_SPAN)]
    + [("bollinger", w) for w in (1, 2, IND_MAX_WINDOW)]
    + [("stochastic", p) for p in ((1, 3), (2, 3), (IND_MAX_WINDOW, 3), (14, 1), (14, 2), (14, IND_MAX_WINDOW),
                                   (IND_MAX_WINDOW, IND_MAX_WINDOW))]
    + [("williams_r", w) for w in (1, 2, IND_MAX_WINDOW)]
    + [("ichimoku", (w, 26, 52)) for w in (1, 2, IND_MAX_WINDOW)]
    + [("ichimoku", (9, w, 52)) for w in (1, 2, IND_MAX_WINDOW)]
    + [("ichimoku", (9, 26, w)) for w in (1, 2, IND_MAX_WINDOW)]
    + [("vwap", w) for w in (1, 2, IND_MAX_WINDOW)]
)


@pytest.mark.parametrize("entry,p", BOUNDS, ids=[f"{e}-{p}" for e, p in BOUNDS])
def test_window_bounds_at_tile_seams(torch_cuda, entry, p):
    """w = 1, 2 and the largest window each entry point accepts, on series that end just before, at and after the window
    (the warm-up NaN / 0 edge, the ATR seed bar), on either side of a tile seam, and one tile past the whole halo (a tile
    whose warm-up crosses many tiles).  NaN pattern exact, values within the bounds of the price-scale test."""
    torch = torch_cuda
    w = max(p) if isinstance(p, (list, tuple)) else p
    tile = RSI_TILE if entry == "rsi" else IND_TILE
    halo = _seam_halo(entry, p)
    ns = sorted({n for n in (w - 2, w - 1, w, tile - 1, tile, tile + 1, halo + tile + 1) if n >= 1})
    for N in ns:
        data = _two_scales(N, seed=N)
        got = _gpu(entry, p, _dev(torch, data))
        _check_against_ref(entry, p, data, got, (entry, p, "N", N))


# ---------------------------------------------------------------------------------------------------------------------
# 4. wide banks and refusals
# ---------------------------------------------------------------------------------------------------------------------
def _spread(bound, P, seed):
    """P windows over [1, bound]: both ends, duplicates of each, the rest drawn at random (one of them twice)."""
    rng = np.random.default_rng(seed)
    rest = [int(x) for x in rng.integers(1, bound + 1, P - 6)]
    return [1, 1, 2, bound, bound] + rest + [rest[0]]


@pytest.mark.parametrize("entry,bound,P,N", [("ema", IND_MAX_WINDOW, IND_MAX_P, 24001),
                                             ("sma", IND_MAX_WINDOW, IND_MAX_P, 24001),
                                             ("atr", ATR_MAX_WINDOW, IND_MAX_P, 12001),
                                             ("rsi", RSI_TILE, RSI_MAX_P, 20001)])
def test_wide_bank_rows_equal_each_window_alone(torch_cuda, entry, bound, P, N):
    """A full bank (one warp walks several windows): each row equals that window computed alone, bitwise, and the float64
    reference; a permuted bank gives the permuted rows, bitwise.  (The recurrences start each window's scan at its own halo;
    the SMA bank's staged span follows its longest window, but its fp64 prefix sums of fp32 offsets are exact.)"""
    torch = torch_cuda
    windows = _spread(bound, P, seed=P + bound)
    assert len(windows) == P
    data = _two_scales(N, seed=3)
    t = _dev(torch, data)
    bank = _gpu(entry, windows, t)[entry]
    assert bank.shape == (2, P, N)
    alone = {}
    for w in sorted(set(windows)):
        alone[w] = _gpu(entry, [w], t)[entry][:, 0]
    for i, w in enumerate(windows):
        assert _same_bits(bank[:, i], alone[w]), (entry, "row", i, "window", w)
    perm = np.random.default_rng(1).permutation(P)
    permuted = _gpu(entry, [windows[j] for j in perm], t)[entry]
    assert _same_bits(permuted, bank[:, perm]), (entry, "permuted bank")
    uniq = sorted(set(windows))
    _check_against_ref(entry, uniq, data, {entry: np.stack([alone[w] for w in uniq], axis=1)}, (entry, "bank"))


def test_each_bound_is_accepted_at_the_limit_and_refused_past_it(torch_cuda):
    """At the bound the call runs; one past it, or a zero window / empty bank, it is refused with the status its entry
    point's check names.  (The window bounds' values are checked against the reference in test_window_bounds_at_tile_seams.)"""
    torch = torch_cuda
    from ai_crypto_trader_b200 import _lib, indicators as ind
    from ai_crypto_trader_b200._lib import B200btError
    from ai_crypto_trader_b200.sweep import rsi_bank
    N = 300
    o, h, l, c, v = _dev(torch, _ohlcv(2, N))

    def refused(status, fn, *a, **kw):
        with pytest.raises(B200btError) as e:
            fn(*a, **kw)
        assert e.value.status == status, (fn.__name__, a[-2:], kw, e.value)

    # banks: windows per call and window length
    for name, fn, args, bound in (("ema_bank", ind.ema_bank, (c,), IND_MAX_WINDOW),
                                  ("sma_bank", ind.sma_bank, (c,), IND_MAX_WINDOW),
                                  ("atr_bank", ind.atr_bank, (h, l, c), ATR_MAX_WINDOW)):
        assert fn(*args, [bound] * IND_MAX_P).shape == (2, IND_MAX_P, N), name
        refused(ELIMIT, fn, *args, [bound] * (IND_MAX_P + 1))
        refused(ELIMIT, fn, *args, [bound + 1])
        refused(ELIMIT, fn, *args, [0])
    refused(ELIMIT, ind.atr_bank, h, l, c, [IND_MAX_WINDOW])
    assert rsi_bank(c, [RSI_TILE] * RSI_MAX_P).shape == (2, RSI_MAX_P, N)
    refused(ELIMIT, rsi_bank, c, [14] * (RSI_MAX_P + 1))
    refused(ELIMIT, rsi_bank, c, [RSI_TILE + 1])
    refused(ELIMIT, rsi_bank, c, [0])
    # empty banks, through the C entry points with a real output buffer (an empty tensor has no storage, and the
    # null-pointer check would answer first): the bank checks refuse P = 0 with ELIMIT, the RSI bank's size check with EINVAL
    buf = torch.empty((2, 1, N), dtype=torch.float32, device="cuda")
    no_windows = (ctypes.c_int * 1)(14)
    for fn, ins in (("b200bt_ema_bank", (c,)), ("b200bt_sma_bank", (c,)), ("b200bt_atr_bank", (h, l, c))):
        refused(ELIMIT, _lib.call, fn, *[x.data_ptr() for x in ins], 2, N, N, no_windows, 0, buf.data_ptr(),
                _lib.current_stream())
    refused(EINVAL, _lib.call, "b200bt_rsi_bank", c.data_ptr(), 2, N, N, no_windows, 0, 0, buf.data_ptr(),
            _lib.current_stream())
    # MACD: each span at 512 runs, 513 and 0 are refused
    for i in range(3):
        spans = [12, 26, 9]
        spans[i] = MACD_MAX_SPAN
        ind.macd(c, *spans)
        spans[i] = MACD_MAX_SPAN + 1
        refused(ELIMIT, ind.macd, c, *spans)
        spans[i] = 0
        refused(ELIMIT, ind.macd, c, *spans)
    # single-window entry points at 1024, 1025 and 0
    for W, ok in ((IND_MAX_WINDOW, True), (IND_MAX_WINDOW + 1, False), (0, False)):
        calls = [(ind.bollinger, (c, W)), (ind.stochastic, (h, l, c, W, 3)), (ind.stochastic, (h, l, c, 14, W)),
                 (ind.williams_r, (h, l, c, W)), (ind.ichimoku, (h, l, W, 26, 52)), (ind.ichimoku, (h, l, 9, W, 52)),
                 (ind.ichimoku, (h, l, 9, 26, W)), (ind.vwap, (h, l, c, v, W))]
        for fn, a in calls:
            if ok:
                fn(*a)
            else:
                refused(ELIMIT, fn, *a)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# 5. layout independence
# ---------------------------------------------------------------------------------------------------------------------
def test_symbols_of_every_price_scale_in_one_call_equal_each_symbol_alone(torch_cuda):
    """33 symbols whose prices run from 1e-5 to 1e5 in one call: every row equals that symbol computed alone, bitwise."""
    torch = torch_cuda
    S, N = 33, 5001
    data = _ohlcv(S, N, seed=9, scales=[10.0 ** (-7 + 10 * s / (S - 1)) for s in range(S)])   # closes ~1e-5 .. ~1e5
    assert data[3, 0].min() < 2e-5 and data[3, -1].max() > 5e4
    together = _all_outputs(torch, data)
    for s in range(S):
        alone = _all_outputs(torch, np.ascontiguousarray(data[:, s:s + 1]))
        for key, x in alone.items():
            assert _same_bits(together[key][s:s + 1], x), (s, key)


def _strided(torch, x, pad, offset):
    """numpy [S][N] -> device view [S][N] with row stride N + pad, starting `offset` floats into a NaN-filled buffer."""
    S, N = x.shape
    buf = torch.full((offset + S * (N + pad),), float("nan"), dtype=torch.float32, device="cuda")
    view = buf[offset:].view(S, N + pad)[:, :N]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    return view


def _call_outputs(t, entries=None):
    out = {}
    for i, (entry, p) in enumerate(CALLS):
        if entries is None or entry in entries:
            for name, x in _gpu(entry, p, t).items():
                out[(i, name)] = x
    return out


def test_padded_rows_with_an_odd_stride_off_alignment_equal_contiguous_rows(torch_cuda):
    """Rows of a padded buffer (row stride N + 5, first row one float into the buffer: rows start off 16-byte alignment)
    give the same outputs as contiguous rows, bitwise."""
    torch = torch_cuda
    from ai_crypto_trader_b200 import _lib
    data = _two_scales(6001, seed=4)
    dense = _call_outputs(_dev(torch, data))
    t = [_strided(torch, data[f], pad=5, offset=1) for f in range(5)]
    assert _lib.ld(t[3]) == 6006 and t[3].data_ptr() % 16 != 0
    padded = _call_outputs(t)
    for key, x in dense.items():
        assert _same_bits(padded[key], x), key


def test_inputs_with_different_row_strides_equal_contiguous_rows(torch_cuda):
    """high, low, close and volume with four different row strides give the outputs of contiguous rows, bitwise: the
    wrappers copy such inputs to contiguous rows, since each kernel reads all of a call's inputs with one row stride.
    (Close is the densest and high denser than low, so a kernel that used close's stride for every input, or high's for
    low, would read other symbols' bars inside the buffers rather than past them.)"""
    torch = torch_cuda
    from ai_crypto_trader_b200 import _lib
    S, N = 4, 5001
    data = _ohlcv(S, N, seed=8, scales=[0.5, 1.0, 3.0, 7.0])
    several = ("atr", "stochastic", "williams_r", "ichimoku", "vwap")     # the entry points that read more than one row
    dense = _call_outputs(_dev(torch, data), several)
    o = _strided(torch, data[0], pad=11, offset=0)
    h = _strided(torch, data[1], pad=3, offset=1)
    l = _strided(torch, data[2], pad=5, offset=2)
    c = torch.from_numpy(np.ascontiguousarray(data[3])).cuda()
    v = _strided(torch, data[4], pad=N + 1, offset=3)
    assert len({_lib.ld(x) for x in (h, l, c, v)}) == 4
    mixed = _call_outputs([o, h, l, c, v], several)
    for key, x in dense.items():
        assert _same_bits(mixed[key], x), (CALLS[key[0]], key[1], "rows that differ:",
                                           [s for s in range(S) if not _same_bits(mixed[key][s], x[s])])


@pytest.mark.parametrize("N", [8192, 8195])
def test_rsi_bank_into_an_output_off_alignment(torch_cuda, N):
    """rsi_bank into a caller's `out` that starts one float off 16-byte alignment (the kernel's scalar store path) equals
    the aligned call, bitwise, with and without the NaN policy."""
    torch = torch_cuda
    from ai_crypto_trader_b200.sweep import rsi_bank
    c = _dev(torch, _two_scales(N, seed=2))[3]
    for periods, fill in itertools.product(([1, 2, 5, 14, 30, 14], [14, 1100, RSI_TILE]), (True, False)):   # halo staged / read
        aligned = rsi_bank(c, periods, fill=fill)
        assert aligned.data_ptr() % 16 == 0
        buf = torch.full((1 + aligned.numel(),), -1.0, dtype=torch.float32, device="cuda")
        out = buf[1:].view(aligned.shape)
        assert rsi_bank(c, periods, fill=fill, out=out) is out
        assert _same_bits(out.cpu().numpy(), aligned.cpu().numpy()), (N, periods, fill)
        assert buf[0].item() == -1.0


def test_rsi_bank_copies_a_time_strided_close_to_contiguous_rows(torch_cuda):
    """rsi_bank(close[:, ::2]) is the bank of every other bar: the wrapper makes a time-strided close contiguous (the
    kernel reads a row's bars as consecutive floats)."""
    torch = torch_cuda
    from ai_crypto_trader_b200.sweep import rsi_bank
    from oracle import indicators_ref as ref
    periods = [2, 14, 30]
    data = _two_scales(10001, seed=6)
    c = _dev(torch, data)[3]
    got = rsi_bank(c[:, ::2], periods).cpu().numpy()
    want = rsi_bank(c[:, ::2].contiguous(), periods).cpu().numpy()
    assert _same_bits(got, want)
    for s in range(2):
        np.testing.assert_allclose(got[s], ref.rsi_bank(data[3, s, ::2], periods), rtol=2e-7, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# 6. the fused analyzer and the entry points run the same tile functions
# ---------------------------------------------------------------------------------------------------------------------
def test_analyzer_columns_equal_the_single_indicator_entry_points(torch_cuda):
    """Over several tiles at both price scales, wherever an entry point's output is defined, the analyzer's column (NaN
    policy applied) is the same bit for bit: sma_20 / 50 / 200 (the bank of those windows stages the analyzer's 199-bar
    span), stoch_k, stoch_d, williams_r, ichimoku_a, ichimoku_b (exact extrema, one walk) and vwap (vwap_tile, same span).
    The other columns differ in their last bits by design: Bollinger's Σd² rounds with the staged span (19 bars alone, 199
    in the analyzer), ATR's and the EMAs' scans start at other bars (sub-tiles, the MACD halo), RSI is another kernel."""
    torch = torch_cuda
    from ai_crypto_trader_b200.indicators import TechnicalAnalyzer
    from ai_crypto_trader_b200.sweep import MarketData
    N = 3 * IND_TILE + 777
    data = _two_scales(N, seed=12)
    t = _dev(torch, data)
    cols = {name: x.cpu().numpy() for name, x in TechnicalAnalyzer(MarketData(data)).data.items()}
    sma = _gpu("sma", [20, 50, 200], t)["sma"]
    alone = {"sma_20": sma[:, 0], "sma_50": sma[:, 1], "sma_200": sma[:, 2], **_gpu("stochastic", (14, 3), t),
             **_gpu("williams_r", 14, t), **_gpu("ichimoku", (9, 26, 52), t), **_gpu("vwap", 14, t)}
    for name, want in alone.items():
        defined = ~np.isnan(want)
        assert defined.sum() >= 2 * (N - 200), name
        got = cols[name]
        assert _same_bits(got[defined], want[defined]), (name, "bars that differ:",
                                                         np.flatnonzero((got != want) & defined)[:8])
