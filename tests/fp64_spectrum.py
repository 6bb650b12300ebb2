"""Double-precision restatement of the reference's spectrum tick (`WAVSourceGeneric::tick_spectrum`,
src/source_generic.cpp:26-179), the ground truth every spectrum kernel and the oracle are measured against.

Only the arithmetic differs from the engine: the window, slope and roll-off tables are the engine's own float32 tables
(`engine.preview_tables`, bit-exact with the reference's `WAVSource::update`), and gravity is the float32 value
`get_gravity(seconds)` yields (a scalar, or one per tick for TV-exponential smoothing).  Everything else runs in
float64: window multiply, an exact DFT (`numpy.fft.rfft`), |X|·2/Σw, slope, EMA (incl. the fast-peaks rule), dBFS,
the 2 -> 1 channel mix or stereo, volume normalisation and roll-off, with the silence gate / hold and the "not enough
audio" skip (`skip_mask`) restated line by line.
"""
from __future__ import annotations

import numpy as np

TSMOOTH_NONE = 0
ULP = 2.0 ** -23                  # one float32 ulp, relative
DB_LOG_ABS = 6.0206 * 2.0 ** -22  # dB = 6.0206·lg2.approx(x): lg2.approx's absolute error floor, in dB
# |X|·coef below this may come out as an exact zero (DESIGN §2): the kernels square each component with flush-to-zero
# and take sqrt.approx.ftz, so a bin whose re² and im² are both below FLT_MIN reads 0: |X|·coef < sqrt(2·FLT_MIN)
FLUSH = float(np.sqrt(2.0 * np.finfo(np.float32).tiny))
FLOOR_DB = -600.0                 # DB_MIN (+ volume gain): a gated / skipped / flushed value, zero on both sides


def engine_tables(settings: dict | None, channels: int, sample_rate: int = 48000) -> dict:
    """The engine's float32 tables and facts for these settings (no device needed)."""
    from waveform_b200.engine import make_config, preview_tables

    cfg = make_config(settings, sample_rate, channels)
    t = preview_tables(cfg)
    info = t["info"]
    return {
        "cfg": cfg, "N": int(info.fft_size), "B": int(info.bins), "cc": int(info.capture_channels),
        "och": int(info.output_channels), "dch": int(info.display_channels),
        "window_sum": np.float32(info.window_sum), "db_min": float(np.float32(info.db_min)),
        "window": t["window"], "slope": t["slope"], "rolloff": t["rolloff"],
    }


class Fp64Spectrum:
    """One source (m_tsmooth_buf, m_decibels, m_last_silent as the reference keeps them, in float64) fed tick by tick.
    State persists across run() calls, like the engine's per-stream state across process() calls."""

    def __init__(self, settings: dict | None = None, channels: int = 1, sample_rate: int = 48000):
        t = engine_tables(settings, channels, sample_rate)
        c = t["cfg"]
        self.N, self.B, self.cc, self.och, self.dch = t["N"], t["B"], t["cc"], t["och"], t["dch"]
        self.db_min = t["db_min"]
        self.window = t["window"].astype(np.float64) if t["window"].size else None
        self.slope = t["slope"].astype(np.float64) if (c.slope > 0.0 and t["slope"].size) else None
        self.rolloff = t["rolloff"].astype(np.float64) if (c.rolloff_q > 0.0 and c.rolloff_rate > 0.0 and t["rolloff"].size) else None
        self.coef = 2.0 / float(t["window_sum"])
        self.tsmooth = c.tsmoothing != TSMOOTH_NONE
        self.fast_peaks = bool(c.fast_peaks)
        self.stereo = bool(c.stereo)
        self.floor_m10 = float(np.float32(c.floor_db - 10))
        self.normalize = bool(c.normalize_volume)
        self.vol_target, self.max_gain = float(np.float32(c.volume_target)), float(np.float32(c.max_gain))
        self.reset()

    def reset(self):
        self.state = np.zeros((self.cc, self.B))                    # m_tsmooth_buf
        self.decibels = np.full((self.och, self.B), self.db_min)    # m_decibels
        self.last_silent = False                                     # m_last_silent
        # What a float32 implementation cannot do better than, per bin, for compare():
        # db_eps: error budget, in dB, of each m_decibels row: one ulp per float32 rounding of the dB steps (dbfs, volume,
        #   roll-off), and at least DB_LOG_ABS per logarithm (the kernels' documented lg2.approx has an absolute error
        #   floor, which matters near 0 dB).  A row a skipped tick pushes through dbfs() again carries the previous row's
        #   budget along: d(20 log10 x) = 8.686 dx / x.
        # flush: bound on the linear error, at the |X|·coef scale, from magnitudes below FLUSH that come out as exact
        #   zeros (sqrt.approx.ftz), carried through the EMA: state_flush (per capture channel, at the state's scale) and
        #   the display rows.
        self.db_eps = np.zeros((self.och, self.B))
        self.state_flush = np.zeros((self.cc, self.B))
        self.flush = np.zeros((self.dch, self.B))
        # per output bin, the linear factor slope, volume and roll-off applied to |X|·coef in the last computed row
        self.weight = np.ones((self.dch, self.B))

    def dbfs(self, x):
        x = np.asarray(x, dtype=np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(x > 0.0, 20.0 * np.log10(np.where(x > 0.0, x, 1.0)), self.db_min)

    def magnitudes(self, frame):
        """|X_k|·2/Σw, k < N/2, of one float32 frame, in float64."""
        x = np.asarray(frame, dtype=np.float64)
        if self.window is not None:
            x = x * self.window
        return np.abs(np.fft.rfft(x)[: self.B]) * self.coef

    @staticmethod
    def _log_eps(d):
        return np.maximum(np.abs(d) * ULP, DB_LOG_ABS)

    def _stale_eps(self, x, eps):
        """Budget carried by dbfs(x) of a stale dB value x whose own budget is eps."""
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(x > 0.0, 8.686 * eps / np.where(x > 0.0, x, 1.0), 0.0)

    def tick(self, frames, g, input_rms=0.0):
        """frames: one float32 array of N samples per capture channel, or None where the tick has not enough audio.
        g: the float32 gravity of this tick.  Returns (dB rows [dch, B] float64, m_last_silent)."""
        g = np.float32(g)
        g1, g2 = float(g), float(np.float32(1.0) - g)     # the reference's g and g2 = 1.0f - g
        silent_channels = 0
        fresh = [False] * self.och
        fl = np.zeros((self.och, self.B))
        slope = self.slope if self.slope is not None else 1.0
        for ch in range(self.cc):
            frame = frames[ch]
            if frame is None:
                continue
            silent = not np.any(frame != 0.0)
            if not silent:
                self.last_silent = False
            if silent:
                if self.last_silent:
                    continue
                if not np.any(self.decibels[ch if self.stereo else 0] > self.floor_m10):
                    silent_channels += 1
                    if silent_channels >= self.cc:
                        self.last_silent = True
                    continue
            raw = self.magnitudes(frame)
            flushed = np.where(raw < FLUSH, raw, 0.0) * slope
            mag = raw * slope
            if self.tsmooth:
                old = self.state[ch]
                if self.fast_peaks:
                    old = np.maximum(mag, old)
                mag = g1 * old + g2 * mag
                self.state[ch] = mag
                self.state_flush[ch] = g1 * self.state_flush[ch] + flushed
            else:
                self.state_flush[ch] = flushed
            self.decibels[ch] = mag
            fresh[ch] = True
            fl[ch] = self.state_flush[ch]
        if not self.last_silent:
            prev = self.decibels.copy()
            if self.och > self.cc:
                self.decibels[1] = self.decibels[0]
                fresh[1], fl[1] = fresh[0], fl[0]
                self.db_eps[1] = self.db_eps[0]
            if self.stereo:
                self.decibels[:2] = self.dbfs(self.decibels[:2])
                for c in range(2):
                    e = self._log_eps(self.decibels[c])
                    self.db_eps[c] = e if fresh[c] else e + self._stale_eps(prev[c], self.db_eps[c])
            elif self.cc > 1:
                avg = (self.decibels[0] + self.decibels[1]) * 0.5
                self.decibels[0] = self.dbfs(avg)
                e = self._log_eps(self.decibels[0])
                stale = sum(self.db_eps[c] * 0.5 for c in range(2) if not fresh[c])
                self.db_eps[0] = e + (self._stale_eps(avg, stale) if not all(fresh[:2]) else 0.0)
                fl[0] = (fl[0] + fl[1]) * 0.5
            else:
                self.decibels[0] = self.dbfs(self.decibels[0])
                e = self._log_eps(self.decibels[0])
                self.db_eps[0] = e if fresh[0] else e + self._stale_eps(prev[0], self.db_eps[0])
            d, eps = self.decibels[: self.dch], self.db_eps[: self.dch]
            self.weight = np.ones((self.dch, self.B)) if self.slope is None else np.tile(self.slope, (self.dch, 1))
            self.flush = fl[: self.dch] / slope
            if self.normalize:
                rms_db = float(self.dbfs(float(np.float32(input_rms))))
                vc = min(self.vol_target - rms_db, self.max_gain)
                d[:, 1:] += vc
                eps[:, 1:] += float(self._log_eps(rms_db)) + abs(vc) * ULP + np.abs(d[:, 1:]) * ULP
                self.weight[:, 1:] *= 10.0 ** (vc / 20.0)
            if self.rolloff is not None:
                d[:, 1:] = np.maximum(d[:, 1:] - self.rolloff[1:], self.db_min)
                eps[:, 1:] += np.abs(d[:, 1:]) * ULP
                self.weight[:, 1:] *= 10.0 ** (-self.rolloff[1:] / 20.0)
        return self.decibels[: self.dch].copy(), self.last_silent

    def run(self, pcm, n_frames: int, hop: int, gravity, input_rms=None, skip_mask=None) -> dict:
        """pcm [cc, samples] float32; gravity: a float32 scalar or one per tick; input_rms / skip_mask: one per tick.
        Returns dB rows [T, dch, B], silent flags [T], the linear EMA state [cc, B] after the last tick and its flush
        bound, and per tick db_eps, flush and weight [T, dch, B] (see reset())."""
        pcm = np.atleast_2d(np.asarray(pcm, dtype=np.float32))
        gs = np.broadcast_to(np.asarray(gravity, dtype=np.float32), (n_frames,))
        db = np.empty((n_frames, self.dch, self.B))
        db_eps, flush, weight = np.empty_like(db), np.empty_like(db), np.empty_like(db)
        silent = np.zeros(n_frames, dtype=bool)
        for t in range(n_frames):
            skip = skip_mask is not None and bool(skip_mask[t])
            frames = [None if skip else pcm[ch, t * hop: t * hop + self.N] for ch in range(self.cc)]
            rms = 0.0 if input_rms is None else input_rms[t]
            db[t], silent[t] = self.tick(frames, gs[t], rms)
            db_eps[t], flush[t], weight[t] = self.db_eps[: self.dch], self.flush, self.weight
        return {"db": db, "silent": silent, "tsmooth": self.state.copy(), "tsmooth_flush": self.state_flush.copy(),
                "db_eps": db_eps, "flush": flush, "weight": weight}


def lin(db):
    return np.power(10.0, np.asarray(db, dtype=np.float64) / 20.0)


def normwise_vs_truth(got_db, truth_db, db_min):
    """Per-frame normwise error max|lin(got) - lin(truth)| / max lin(truth) over the frame (the last axis and the display
    channel axis before it), in the linear domain; DB_MIN counts as 0 on both sides.  Returns [frames...] float64."""
    g, r = lin(got_db), lin(truth_db)
    g[np.asarray(got_db) <= db_min + 1e-3] = 0.0
    r[np.asarray(truth_db) <= db_min + 1e-3] = 0.0
    peak = np.maximum(r.max(axis=(-1, -2)), 1e-300)
    return np.abs(g - r).max(axis=(-1, -2)) / peak


def compare(got_db, tr, db_min):
    """Per-frame normwise error [frames] of float32 dB rows against a run() result, and whether any bin reports DB_MIN
    where float64 puts it at or above FLUSH and above the frame's float32 resolution.

    Both rows are divided by the linear factor slope, volume and roll-off applied to each bin (tr["weight"]), so that the
    error is measured at the |X|·coef scale an FFT's rounding error follows: roll-off and slope can take a low-frequency
    peak down by tens of dB, and any float32 FFT's error against the weighted peak grows by as much.  Each bin's
    difference then loses what no float32 implementation with the documented approximations can avoid: the dB budget
    tr["db_eps"] and the carried flush bound tr["flush"]."""
    g, r = lin(got_db) / tr["weight"], lin(tr["db"]) / tr["weight"]
    g[np.asarray(got_db) <= FLOOR_DB] = 0.0
    r[np.asarray(tr["db"]) <= FLOOR_DB] = 0.0
    db_tol = r * (np.log(10.0) / 20.0) * tr["db_eps"]
    d = np.maximum(np.abs(g - r) - tr["flush"] - db_tol, 0.0)
    peak = r.max(axis=(-1, -2))
    err = np.where(peak > 0, d.max(axis=(-1, -2)) / np.maximum(peak, 1e-300), 0.0)
    above = (r >= FLUSH) & (r >= 1e-6 * peak[..., None, None])
    bad_floor = (np.asarray(got_db) <= db_min + 1e-3) & above
    return err, bool(bad_floor.any())
