"""ctypes binding of libwfstft.so (include/wfstft.h) — the product's C-ABI, nothing else.

This module deliberately contains no DSP: every number comes out of the CUDA library.  If the
library is missing, or there is no sm_90 device, construction fails loudly (no CPU fallback).

Settings use the reference plugin's own setting keys (/root/reference/src/settings.hpp:29-135), so a
caller (or a test) configures the engine exactly as it would configure the OBS source:

    eng = Engine({"fft_size": 2048, "window": "hann", "temporal_smoothing": "exp_moving_avg"},
                 channels=1, max_streams=256)
    out = eng.process(pcm, n_frames=256, hop=2048)     # pcm: numpy (host) or torch.cuda tensor (device)
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
# WF_LIB_PATH: development knob to A/B a differently compiled build of the SAME library (never a fallback)
LIB_PATH = Path(os.environ["WF_LIB_PATH"]) if os.environ.get("WF_LIB_PATH") else _HERE / "lib" / "libwfstft.so"

WF_OK = 0
WF_ERR_INVALID_ARG = -1
WF_ERR_UNSUPPORTED_FFT_SIZE = -2
WF_ERR_CUDA = -3
WF_ERR_NO_DEVICE = -4
WF_ERR_OOM = -5
WF_ERR_CAPACITY = -6
WF_ERR_ABI = -7

WINDOWS = {"none": 0, "hann": 1, "hamming": 2, "blackman": 3, "blackman_harris": 4, "power_of_sine": 5}
INTERPS = {"point": 0, "lanczos": 1, "catmull_rom": 2}
FILTERS = {"none": 0, "gauss": 1}
TSMOOTH = {"none": 0, "exp_moving_avg": 1, "tv_exp_moving_avg": 2}
DISPLAYS = {"curve": 0, "bars": 1, "stepped_bars": 1}

TABLE_WINDOW, TABLE_SLOPE, TABLE_ROLLOFF, TABLE_INTERP_INDICES, TABLE_INTERP_WEIGHTS, TABLE_BAND_WIDTHS, TABLE_GAUSS = range(7)

EXPORTS = [
    "wf_abi_version", "wf_strerror", "wf_last_error", "wf_config_init", "wf_create", "wf_destroy", "wf_get_info",
    "wf_get_table", "wf_gravity", "wf_process", "wf_process_async", "wf_synchronize", "wf_reset_state",
    "wf_get_state", "wf_set_state", "wf_get_ring", "wf_set_ring", "wf_peak_normalize", "wf_launch_count", "wf_last_kernel_ms", "wf_last_kernel_name",
    "wf_host_alloc", "wf_host_free", "wf_preview_table", "wf_render",
    "wf_meter_config_init", "wf_meter_create", "wf_meter_destroy", "wf_meter_last_error", "wf_meter_window",
    "wf_meter_process", "wf_meter_process_async", "wf_meter_reset", "wf_meter_get_state", "wf_meter_set_state",
    "wf_meter_launch_count", "wf_meter_last_kernel_ms",
    "wf_wave_config_init", "wf_wave_create", "wf_wave_create_with_clock", "wf_wave_destroy", "wf_wave_last_error",
    "wf_wave_process", "wf_wave_process_async", "wf_wave_reset", "wf_wave_get_state", "wf_wave_set_state",
    "wf_wave_get_clock", "wf_wave_set_clock", "wf_wave_launch_count", "wf_wave_last_kernel_ms",
    "wf_wave_preview_plan", "wf_wave_preview_table",
]

METER_PEAK, METER_RMS, METER_INPUT_RMS = 0, 1, 2


class WfMeterConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_streams", C.c_int32), ("sample_rate", C.c_uint32),
        ("capture_channels", C.c_int32), ("mode", C.c_int32), ("meter_ms", C.c_int32), ("tsmoothing", C.c_int32),
        ("gravity", C.c_float), ("fast_peaks", C.c_int32), ("floor_db", C.c_int32),
        ("height", C.c_int32), ("ceiling_db", C.c_int32), ("bar_width", C.c_int32), ("rounded_caps", C.c_int32),
        ("min_bar_height", C.c_int32), ("sync_offset_ms", C.c_int32),
    ]


class WfWaveConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_streams", C.c_int32), ("sample_rate", C.c_uint32),
        ("capture_channels", C.c_int32), ("stereo", C.c_int32), ("width", C.c_int32), ("meter_ms", C.c_int32),
        ("normalize_volume", C.c_int32), ("volume_target", C.c_float), ("max_gain", C.c_float),
        ("interp_mode", C.c_int32), ("filter_mode", C.c_int32), ("filter_radius", C.c_float), ("height", C.c_int32),
        ("floor_db", C.c_int32), ("ceiling_db", C.c_int32), ("channel_spacing", C.c_int32), ("sync_offset_ms", C.c_int32),
    ]


class WfWaveBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_ticks", C.c_int32), ("hop", C.c_int32),
        ("pcm", C.c_void_p), ("stream_stride", C.c_int64), ("channel_stride", C.c_int64),
        ("input_rms", C.c_void_p), ("out", C.c_void_p), ("out_silent", C.c_void_p),
        ("out_points", C.c_void_p), ("out_pixels", C.c_void_p), ("out_min", C.c_void_p),
        ("pcm_format", C.c_int32),
    ]


class WfWaveClock(C.Structure):
    """wf_wave_clock: the engine-wide clock of tick_waveform (WaveEngine.get_clock / set_clock)."""
    _fields_ = [("clock_ns", C.c_uint64), ("audio_ts", C.c_uint64), ("waveform_ts", C.c_uint64), ("buffered", C.c_uint64)]


class WfMeterBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_ticks", C.c_int32), ("hop", C.c_int32),
        ("first_stream", C.c_int32), ("seconds", C.c_float),
        ("pcm", C.c_void_p), ("stream_stride", C.c_int64), ("channel_stride", C.c_int64),
        ("out_db", C.c_void_p), ("out_lin", C.c_void_p), ("out_silent", C.c_void_p),
        ("out_pixels", C.c_void_p), ("out_min", C.c_void_p),
        ("pcm_format", C.c_int32),
    ]


class WfConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_streams", C.c_int32),
        ("sample_rate", C.c_uint32), ("capture_channels", C.c_int32), ("fft_size", C.c_int32),
        ("window", C.c_int32), ("sine_exponent", C.c_int32), ("tsmoothing", C.c_int32),
        ("gravity", C.c_float), ("fast_peaks", C.c_int32), ("slope", C.c_float),
        ("rolloff_q", C.c_float), ("rolloff_rate", C.c_float),
        ("cutoff_low", C.c_int32), ("cutoff_high", C.c_int32),
        ("floor_db", C.c_int32), ("ceiling_db", C.c_int32), ("stereo", C.c_int32),
        ("normalize_volume", C.c_int32), ("volume_target", C.c_float), ("max_gain", C.c_float),
        ("silence_gate", C.c_int32), ("display_mode", C.c_int32),
        ("width", C.c_int32), ("bar_width", C.c_int32), ("bar_gap", C.c_int32),
        ("log_scale", C.c_int32), ("mirror_freq_axis", C.c_int32),
        ("interp_mode", C.c_int32), ("filter_mode", C.c_int32), ("filter_radius", C.c_float),
        ("height", C.c_int32), ("channel_spacing", C.c_int32), ("rounded_caps", C.c_int32), ("min_bar_height", C.c_int32),
        ("sync_offset_ms", C.c_int32),
    ]


class WfInfo(C.Structure):
    _fields_ = [
        ("fft_size", C.c_int32), ("bins", C.c_int32), ("capture_channels", C.c_int32),
        ("output_channels", C.c_int32), ("display_channels", C.c_int32), ("num_points", C.c_int32),
        ("num_bars", C.c_int32), ("interp_taps", C.c_int32), ("n_interp_indices", C.c_int32),
        ("window_sum", C.c_float), ("db_min", C.c_float), ("device", C.c_int32), ("sm_count", C.c_int32),
    ]


class WfBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_frames", C.c_int32), ("hop", C.c_int32),
        ("first_stream", C.c_int32), ("seconds", C.c_float),
        ("pcm", C.c_void_p), ("stream_stride", C.c_int64), ("channel_stride", C.c_int64),
        ("input_rms", C.c_void_p), ("skip_mask", C.c_void_p),
        ("out_db", C.c_void_p), ("out_points", C.c_void_p), ("out_silent", C.c_void_p), ("out_peak", C.c_void_p),
        ("out_pixels", C.c_void_p), ("out_min", C.c_void_p), ("frame_seconds", C.c_void_p),
        ("pcm_format", C.c_int32),
    ]

    # wf_batch.capture_ring fills what was the struct's tail padding, so sizeof(wf_batch) is unchanged: it is reached as a
    # property over those 4 bytes, and the declared fields stay those of the previous header (whose size is the same)
    @property
    def capture_ring(self) -> int:
        return C.c_uint32.from_buffer(self, type(self).pcm_format.offset + 4).value

    @capture_ring.setter
    def capture_ring(self, v: int):
        C.c_uint32.from_buffer(self, type(self).pcm_format.offset + 4).value = v


# wf_pcm_format: the sample type of wf_batch.pcm, wf_meter_batch.pcm and wf_wave_batch.pcm
PCM_F32, PCM_S16 = 0, 1
# wf_batch.capture_ring of a capture-ring call (WF_CAPTURE_RING)
CAPTURE_RING = 0x676E6972
_PCM_FORMATS = {"f32": PCM_F32, "s16": PCM_S16}


def _pcm_format(name) -> int:
    if name not in _PCM_FORMATS:
        raise ValueError(f"pcm_format must be 'f32' or 's16', got {name!r}")
    return _PCM_FORMATS[name]


class WfRenderBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_frames", C.c_int32),
        ("db", C.c_void_p), ("peak", C.c_void_p), ("target_db", C.c_float), ("max_gain", C.c_float),
        ("write_db", C.c_int32), ("out_points", C.c_void_p), ("out_pixels", C.c_void_p), ("out_min", C.c_void_p),
    ]


class WfError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"libwfstft status {status}: {msg}")
        self.status = status


_lib = None


def load_library():
    """Load libwfstft.so; raises if it has not been built (there is no fallback path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise FileNotFoundError(
            f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C waveform_b200/csrc`.  The engine has no CPU fallback.")
    L = C.CDLL(str(LIB_PATH))
    vp = C.c_void_p
    L.wf_abi_version.restype = C.c_int
    L.wf_strerror.restype = C.c_char_p
    L.wf_strerror.argtypes = [C.c_int]
    L.wf_last_error.restype = C.c_char_p
    L.wf_last_error.argtypes = [vp]
    L.wf_config_init.argtypes = [C.POINTER(WfConfig)]
    L.wf_create.argtypes = [C.POINTER(WfConfig), C.POINTER(vp)]
    L.wf_destroy.argtypes = [vp]
    L.wf_get_info.argtypes = [vp, C.POINTER(WfInfo)]
    L.wf_get_table.restype = C.c_int64
    L.wf_get_table.argtypes = [vp, C.c_int, vp, C.c_int64]
    L.wf_preview_table.restype = C.c_int64
    L.wf_preview_table.argtypes = [C.POINTER(WfConfig), C.c_int, vp, C.c_int64, C.POINTER(WfInfo)]
    L.wf_gravity.restype = C.c_float
    L.wf_gravity.argtypes = [vp, C.c_float]
    L.wf_process.argtypes = [vp, C.POINTER(WfBatch)]
    L.wf_process_async.argtypes = [vp, C.POINTER(WfBatch), vp]
    L.wf_synchronize.argtypes = [vp]
    L.wf_reset_state.argtypes = [vp, C.c_int32, C.c_int32]
    L.wf_get_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.wf_set_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.wf_get_ring.argtypes = [vp, C.c_int32, C.c_int32, vp]
    L.wf_set_ring.argtypes = [vp, C.c_int32, C.c_int32, vp]
    L.wf_peak_normalize.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_float, C.c_float, vp]
    L.wf_render.argtypes = [vp, C.POINTER(WfRenderBatch), vp]
    L.wf_launch_count.restype = C.c_int64
    L.wf_launch_count.argtypes = [vp]
    L.wf_last_kernel_ms.restype = C.c_float
    L.wf_last_kernel_ms.argtypes = [vp]
    L.wf_host_alloc.restype = C.c_void_p
    L.wf_host_alloc.argtypes = [C.c_size_t]
    L.wf_host_free.argtypes = [vp]
    L.wf_last_kernel_name.restype = C.c_char_p
    L.wf_last_kernel_name.argtypes = [vp]
    L.wf_meter_config_init.argtypes = [C.POINTER(WfMeterConfig)]
    L.wf_meter_create.argtypes = [C.POINTER(WfMeterConfig), C.POINTER(vp)]
    L.wf_meter_destroy.argtypes = [vp]
    L.wf_meter_last_error.restype = C.c_char_p
    L.wf_meter_last_error.argtypes = [vp]
    L.wf_meter_window.restype = C.c_int32
    L.wf_meter_window.argtypes = [vp]
    L.wf_meter_process.argtypes = [vp, C.POINTER(WfMeterBatch)]
    L.wf_meter_process_async.argtypes = [vp, C.POINTER(WfMeterBatch), vp]
    L.wf_meter_reset.argtypes = [vp, C.c_int32, C.c_int32]
    L.wf_meter_get_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
    L.wf_meter_set_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
    L.wf_meter_launch_count.restype = C.c_int64
    L.wf_meter_launch_count.argtypes = [vp]
    L.wf_meter_last_kernel_ms.restype = C.c_float
    L.wf_meter_last_kernel_ms.argtypes = [vp]
    L.wf_wave_config_init.argtypes = [C.POINTER(WfWaveConfig)]
    L.wf_wave_create.argtypes = [C.POINTER(WfWaveConfig), C.POINTER(vp)]
    L.wf_wave_create_with_clock.argtypes = [C.POINTER(WfWaveConfig), C.c_int32, C.POINTER(vp)]
    L.wf_wave_destroy.argtypes = [vp]
    L.wf_wave_last_error.restype = C.c_char_p
    L.wf_wave_last_error.argtypes = [vp]
    L.wf_wave_process.argtypes = [vp, C.POINTER(WfWaveBatch)]
    L.wf_wave_process_async.argtypes = [vp, C.POINTER(WfWaveBatch), vp]
    L.wf_wave_reset.argtypes = [vp]
    L.wf_wave_get_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.wf_wave_set_state.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.wf_wave_get_clock.argtypes = [vp, C.POINTER(WfWaveClock)]
    L.wf_wave_set_clock.argtypes = [vp, C.POINTER(WfWaveClock)]
    L.wf_wave_launch_count.restype = C.c_int64
    L.wf_wave_launch_count.argtypes = [vp]
    L.wf_wave_last_kernel_ms.restype = C.c_float
    L.wf_wave_last_kernel_ms.argtypes = [vp]
    L.wf_wave_preview_plan.restype = C.c_int64
    L.wf_wave_preview_plan.argtypes = [C.POINTER(WfWaveConfig), C.c_int32, C.c_int32, vp, vp, C.c_int64]
    L.wf_wave_preview_table.restype = C.c_int64
    L.wf_wave_preview_table.argtypes = [C.POINTER(WfWaveConfig), C.c_int, vp, C.c_int64]
    _lib = L
    return L


def make_config(settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                device: int = -1) -> WfConfig:
    """Reference setting keys -> wf_config (what WAVSource::get_settings does, src/source.cpp:501-674)."""
    L = load_library()
    c = WfConfig()
    L.wf_config_init(C.byref(c))
    c.device = device
    c.max_streams = max_streams
    c.sample_rate = sample_rate
    s = dict(settings or {})
    mode = s.pop("channel_mode", "mono")
    c.stereo = int(mode == "stereo")
    # m_capture_channels = min(channels, 2), or 1 in single-channel mode (src/source.cpp:1089-1101)
    c.capture_channels = min(channels, 2) if mode != "single" else min(channels, 1)
    simple = {
        "fft_size": "fft_size", "sine_exponent": "sine_exponent", "gravity": "gravity", "fast_peaks": "fast_peaks",
        "slope": "slope", "rolloff_q": "rolloff_q", "rolloff_rate": "rolloff_rate", "cutoff_low": "cutoff_low",
        "cutoff_high": "cutoff_high", "floor": "floor_db", "ceiling": "ceiling_db",
        "normalize_volume": "normalize_volume", "volume_target": "volume_target", "max_gain": "max_gain",
        "width": "width", "bar_width": "bar_width", "bar_gap": "bar_gap", "log_scale": "log_scale",
        "mirror_freq_axis": "mirror_freq_axis", "filter_radius": "filter_radius", "silence_gate": "silence_gate",
        "height": "height", "channel_spacing": "channel_spacing", "rounded_caps": "rounded_caps",
        "min_bar_height": "min_bar_height", "audio_sync_offset": "sync_offset_ms",
    }
    enums = {"window": ("window", WINDOWS), "interp_mode": ("interp_mode", INTERPS),
             "filter_mode": ("filter_mode", FILTERS), "temporal_smoothing": ("tsmoothing", TSMOOTH),
             "display_mode": ("display_mode", DISPLAYS)}
    for k, v in s.items():
        if k in simple:
            field = simple[k]
            cur = getattr(c, field)
            setattr(c, field, float(v) if isinstance(cur, float) else int(v))
        elif k in enums:
            field, table = enums[k]
            if v not in table:
                raise ValueError(f"{k}={v!r} is not a spectrum-mode value")
            setattr(c, field, table[v])
        elif k == "auto_fft_size":
            pass  # display plumbing that stays on the host side of the seam
        else:
            raise KeyError(f"setting {k!r} is outside the spectrum hot path")
    return c


def preview_tables(cfg: WfConfig) -> dict:
    """Host-side tables + derived facts for a config, without a device (wf_preview_table)."""
    L = load_library()
    info = WfInfo()
    out = {}
    names = {TABLE_WINDOW: "window", TABLE_SLOPE: "slope", TABLE_ROLLOFF: "rolloff",
             TABLE_INTERP_INDICES: "interp_indices", TABLE_INTERP_WEIGHTS: "interp_weights",
             TABLE_BAND_WIDTHS: "band_widths", TABLE_GAUSS: "gauss"}
    for which, name in names.items():
        n = L.wf_preview_table(C.byref(cfg), which, None, 0, C.byref(info))
        if n < 0:
            raise WfError(int(n), f"{L.wf_strerror(int(n)).decode()}: {L.wf_last_error(None).decode()}")
        arr = np.zeros(n, dtype=np.int32 if which == TABLE_BAND_WIDTHS else np.float32)
        if n:
            L.wf_preview_table(C.byref(cfg), which, arr.ctypes.data, n, None)
        out[name] = arr
    out["info"] = info
    return out


def _ptr(x):
    """Device or host pointer of a torch tensor / numpy array / None."""
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    return x.ctypes.data


class _Handle:
    """What the three engine handles share: creation, error reporting, release, launch count and kernel time.  `_prefix`
    selects the engine kind's C functions (wf_*, wf_meter_*, wf_wave_*)."""

    _prefix = "wf"

    def _fn(self, name):
        return getattr(self.L, f"{self._prefix}_{name}")

    def _create(self, cfg, create="create", *args):
        """`create`: the C function (after the prefix) that makes the handle from cfg, `args` and the handle's address."""
        self.L = load_library()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self._fn(create)(C.byref(cfg), *args, C.byref(h))
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self._fn('last_error')(None).decode()}")
        self.h = h

    def _check(self, rc):
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self._fn('last_error')(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self._fn("destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return int(self._fn("launch_count")(self.h))

    def last_kernel_ms(self) -> float:
        return float(self._fn("last_kernel_ms")(self.h))


def _sync_delay(sample_rate: int, ms: int) -> int:
    """Samples an audio sync offset of `ms` holds back: ns_to_audio_frames(sample_rate, ms * 10**6) for ms > 0, else 0."""
    return sample_rate * ms // 1000 if ms > 0 else 0


def _state_parts(state: dict, parts: dict):
    """The host arrays of a meter / waveform checkpoint for a set call: `parts` maps each key to (per-slot shape, dtype).
    A missing or None part is skipped; the others must be [count, *per-slot shape] with one count, else ValueError (before
    any library call).  Returns (count, {key: contiguous array or None})."""
    out, count = {}, None
    for key, (shape, dtype) in parts.items():
        a = state.get(key)
        if a is not None:
            a = np.ascontiguousarray(a, dtype=dtype)
            if a.ndim != 1 + len(shape) or a.shape[1:] != tuple(shape):
                raise ValueError(f"state[{key!r}] must be [count, {', '.join(map(str, shape))}], got {list(a.shape)}")
            if count is not None and a.shape[0] != count:
                raise ValueError(f"state[{key!r}] holds {a.shape[0]} slots, another part {count}")
            count = a.shape[0]
        out[key] = a
    return (0 if count is None else count), out


class _Inputs:
    """The shared prelude of the engines' process(): `pcm` as [S, channels, samples] (a 2-D array is one stream), checked
    against the engine's channel count and the samples the call needs.  A numpy array becomes contiguous float32 (host
    path); a torch tensor must be a contiguous float32 CUDA tensor (device path), and `stream` is then torch's current
    stream.  new() allocates an output and aux() brings an optional per-tick input to the same side as pcm.
    With s16=True the samples stay int16 as they are: a numpy int16 array or a contiguous int16 CUDA tensor, else ValueError."""

    def __init__(self, pcm, channels: int, need: int, who: str = "engine", s16: bool = False):
        self.is_torch = hasattr(pcm, "data_ptr")
        if pcm.ndim == 2:
            pcm = pcm[None]
        self.S, self.cc, self.ns = pcm.shape
        if self.cc != channels:
            raise ValueError(f"pcm has {self.cc} channels, {who} captures {channels}")
        if self.ns < need:
            raise ValueError(f"need {need} samples per channel, got {self.ns}")
        self.stream = None
        if s16:
            if self.is_torch:
                import torch
                if not (pcm.is_cuda and pcm.dtype == torch.int16 and pcm.is_contiguous()):
                    raise ValueError("pcm_format='s16' needs a contiguous int16 CUDA tensor")
            elif not (isinstance(pcm, np.ndarray) and pcm.dtype == np.int16):
                raise ValueError("pcm_format='s16' needs an int16 numpy array")
        if self.is_torch:
            import torch
            assert s16 or (pcm.is_cuda and pcm.dtype == torch.float32 and pcm.is_contiguous())
            self.f32, self.u8 = torch.float32, torch.uint8
            self.stream = torch.cuda.current_stream(pcm.device).cuda_stream
        else:
            pcm = np.ascontiguousarray(pcm, dtype=np.int16 if s16 else np.float32)
            self.f32, self.u8 = np.float32, np.uint8
        self.pcm = pcm

    def new(self, shape, dtype):
        if self.is_torch:
            import torch
            return torch.empty(shape, dtype=dtype, device=self.pcm.device)
        return np.empty(shape, dtype=dtype)

    def aux(self, x, dtype):
        if x is None:
            return None
        if self.is_torch:
            return x.to(device=self.pcm.device, dtype=dtype).contiguous()
        return np.ascontiguousarray(x, dtype=dtype)


class Engine(_Handle):
    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2,
                 max_streams: int = 1, device: int = -1, config: WfConfig | None = None):
        self._create(config if config is not None else make_config(settings, sample_rate, channels, max_streams, device))
        self.info = WfInfo()
        self._check(self.L.wf_get_info(self.h, C.byref(self.info)))

    # ---- facts ----
    @property
    def fft_size(self):
        return self.info.fft_size

    @property
    def bins(self):
        return self.info.bins

    @property
    def capture_channels(self):
        return self.info.capture_channels

    @property
    def display_channels(self):
        return self.info.display_channels

    @property
    def output_channels(self):
        return self.info.output_channels

    @property
    def num_points(self):
        return self.info.num_points

    @property
    def window_sum(self):
        return self.info.window_sum

    @property
    def db_min(self):
        return self.info.db_min

    def gravity(self, seconds: float) -> float:
        return float(self.L.wf_gravity(self.h, seconds))

    def table(self, which: int):
        n = self.L.wf_get_table(self.h, which, None, 0)
        if n < 0:
            self._check(int(n))
        if n == 0:
            return None
        dtype = np.int32 if which == TABLE_BAND_WIDTHS else np.float32
        out = np.zeros(n, dtype=dtype)
        self.L.wf_get_table(self.h, which, out.ctypes.data, n)
        return out

    def last_kernel_name(self) -> str:
        return self.L.wf_last_kernel_name(self.h).decode()

    # ---- processing ----
    def process_raw(self, pcm_ptr, n_streams, n_frames, hop, stream_stride, channel_stride, *, first_stream=0,
                    seconds=1.0 / 60.0, input_rms=None, skip_mask=None, out_db=None, out_points=None,
                    out_silent=None, out_peak=None, out_pixels=None, out_min=None, stream=None, sync=True,
                    frame_seconds=None, pcm_format="f32", capture_ring=False):
        """Thin wrapper over wf_process / wf_process_async with raw pointers (ints).  pcm_format: "f32" (float samples) or
        "s16" (int16 samples, v * 2**-15); strides and hop count samples either way.  capture_ring: pcm holds only the
        new samples (wf_batch.capture_ring)."""
        b = WfBatch()
        b.struct_size = C.sizeof(WfBatch)
        b.n_streams, b.n_frames, b.hop, b.first_stream = n_streams, n_frames, hop, first_stream
        b.seconds = seconds
        b.pcm = pcm_ptr
        b.stream_stride, b.channel_stride = stream_stride, channel_stride
        b.input_rms, b.skip_mask = input_rms, skip_mask
        b.out_db, b.out_points, b.out_silent, b.out_peak = out_db, out_points, out_silent, out_peak
        b.out_pixels, b.out_min = out_pixels, out_min
        b.frame_seconds = frame_seconds  # host pointer (int) or None
        b.pcm_format = _pcm_format(pcm_format)
        b.capture_ring = CAPTURE_RING if capture_ring else 0
        if sync and stream is None:
            self._check(self.L.wf_process(self.h, C.byref(b)))
        else:
            if stream == 0:
                stream = 1  # the legacy default stream is cudaStreamLegacy (0x1); NULL selects the engine's own stream
            self._check(self.L.wf_process_async(self.h, C.byref(b), stream))

    def process(self, pcm, n_frames: int, hop: int, *, first_stream=0, seconds=1.0 / 60.0, input_rms=None,
                skip_mask=None, want_db=True, want_points=False, want_silent=True, want_peak=False, want_pixels=False,
                frame_seconds=None, pcm_format="f32", capture_ring=False):
        """pcm: [n_streams, capture_channels, samples] float32 — numpy (host path, staged inside the C call)
        or a CUDA torch tensor (device path, outputs are CUDA tensors).  pcm_format="s16": int16 samples instead (an int16
        numpy array or contiguous int16 CUDA tensor), read by the kernels as v * 2**-15; the default converts any numpy
        array to float32 as it is, without scaling.  capture_ring=True: pcm holds only the samples captured since the last
        call, n_frames * hop per channel, and the frames reach back into each stream slot's capture ring (get_ring)."""
        s16 = _pcm_format(pcm_format) == PCM_S16
        need = n_frames * hop if capture_ring else (n_frames - 1) * hop + self.fft_size
        x = _Inputs(pcm, self.capture_channels, need, s16=s16)
        S, cc, ns, mk, f32, u8 = x.S, x.cc, x.ns, x.new, x.f32, x.u8
        input_rms, skip_mask = x.aux(input_rms, f32), x.aux(skip_mask, u8)
        dch, B, P = self.display_channels, self.bins, self.num_points
        out = {}
        if want_db:
            out["db"] = mk((S, n_frames, dch, B), f32)
        if want_points:
            out["points"] = mk((S, n_frames, dch, P), f32)
        if want_silent:
            out["silent"] = mk((S, n_frames), u8)
        if want_peak:
            out["peak"] = mk((n_frames,), f32)
        if want_pixels:
            out["pixels"] = mk((S, n_frames, dch, P), f32)
            out["min"] = mk((S, n_frames, 2), f32)
        # CUDA tensors: launch on torch's CURRENT stream, so the kernel is ordered after whatever produced `pcm` and before
        # whatever consumes the outputs (torch semantics: asynchronous, stream-ordered).  Host arrays: the engine's own
        # stream, synchronised before returning.
        fs = None
        if frame_seconds is not None:  # per-tick `seconds` (always a host array), see wf_batch.frame_seconds
            fs = np.ascontiguousarray(frame_seconds, dtype=np.float32)
            assert fs.shape == (n_frames,)
        self.process_raw(_ptr(x.pcm), S, n_frames, hop, cc * ns, ns, first_stream=first_stream, seconds=seconds,
                         input_rms=_ptr(input_rms), skip_mask=_ptr(skip_mask), out_db=_ptr(out.get("db")),
                         out_points=_ptr(out.get("points")), out_silent=_ptr(out.get("silent")),
                         out_peak=_ptr(out.get("peak")), out_pixels=_ptr(out.get("pixels")), out_min=_ptr(out.get("min")),
                         stream=x.stream, sync=not x.is_torch, frame_seconds=None if fs is None else fs.ctypes.data,
                         pcm_format=pcm_format, capture_ring=capture_ring)
        return out

    def synchronize(self):
        self._check(self.L.wf_synchronize(self.h))

    def reset_state(self, first_stream=0, count=None):
        count = self.cfg.max_streams - first_stream if count is None else count
        self._check(self.L.wf_reset_state(self.h, first_stream, count))

    def get_state(self, first_stream=0, count=None):
        count = self.cfg.max_streams - first_stream if count is None else count
        ts = np.zeros((count, self.capture_channels, self.bins), dtype=np.float32)
        hold = np.zeros((count, self.output_channels, self.bins), dtype=np.float32)
        flags = np.zeros(count, dtype=np.uint8)
        self._check(self.L.wf_get_state(self.h, first_stream, count, ts.ctypes.data, hold.ctypes.data, flags.ctypes.data))
        return {"tsmooth": ts, "hold_db": hold, "flags": flags}

    def set_state(self, state: dict, first_stream=0):
        ts = np.ascontiguousarray(state["tsmooth"], dtype=np.float32) if state.get("tsmooth") is not None else None
        hold = np.ascontiguousarray(state["hold_db"], dtype=np.float32) if state.get("hold_db") is not None else None
        flags = np.ascontiguousarray(state["flags"], dtype=np.uint8) if state.get("flags") is not None else None
        count = len(ts if ts is not None else (hold if hold is not None else flags))
        self._check(self.L.wf_set_state(self.h, first_stream, count, _ptr(ts), _ptr(hold), _ptr(flags)))

    @property
    def sync_delay(self) -> int:
        """Samples the audio sync offset holds back: ns_to_audio_frames(sample_rate, offset) for an offset > 0, else 0."""
        ms = self.cfg.sync_offset_ms if self.cfg.struct_size == C.sizeof(WfConfig) else 0  # the previous size has none
        return _sync_delay(self.cfg.sample_rate, ms)

    def get_ring(self, first_stream=0, count=None):
        """The capture rings of slots [first_stream, first_stream + count): float32
        [count, capture_channels, fft_size + sync_delay], oldest sample first."""
        count = self.cfg.max_streams - first_stream if count is None else count
        ring = np.zeros((count, self.capture_channels, self.fft_size + self.sync_delay), dtype=np.float32)
        self._check(self.L.wf_get_ring(self.h, first_stream, count, ring.ctypes.data))
        return ring

    def set_ring(self, samples, first_stream=0):
        """Replace the capture rings of slots [first_stream, first_stream + len(samples)) with float samples shaped
        [count, capture_channels, fft_size + sync_delay], e.g. to prime a stream with the audio before a cut.  The slots
        then owe no start-up samples to the sync offset."""
        ring = np.ascontiguousarray(samples, dtype=np.float32)
        R = self.fft_size + self.sync_delay
        if ring.ndim != 3 or ring.shape[1:] != (self.capture_channels, R):
            raise ValueError(f"ring samples must be [count, {self.capture_channels}, {R}], got {ring.shape}")
        self._check(self.L.wf_set_ring(self.h, first_stream, ring.shape[0], ring.ctypes.data))

    def peak_normalize(self, data, peak, target_db: float, max_gain: float, stream=None):
        """In-place: data[s, t, ch, k>=1] += min(target_db - peak[t], max_gain).  CUDA tensors run on torch's current
        stream unless `stream` is given (so a preceding all_reduce on that stream is ordered before the pass)."""
        S, T, dch, row = data.shape
        assert dch == self.display_channels
        if stream is None and hasattr(data, "data_ptr") and getattr(data, "is_cuda", False):
            import torch
            stream = torch.cuda.current_stream(data.device).cuda_stream
        if stream == 0:
            stream = 1  # cudaStreamLegacy; NULL would select the engine's private stream
        self._check(self.L.wf_peak_normalize(self.h, _ptr(data), S, T, row, _ptr(peak), target_db, max_gain, stream))

    def render(self, db, peak=None, target_db: float = -3.0, max_gain: float = 30.0, write_db: bool = False,
               want_points: bool = False, want_pixels: bool = False, stream=None):
        """The display stage (wf_render) on dB rows db[S, T, display_channels, bins] — out_db of earlier calls, a numpy array
        (host path, synchronous) or a contiguous float32 CUDA tensor (device path, on torch's current stream unless `stream`
        is given).  With `peak` ([T], numpy or tensor) the cross-channel peak gain min(target_db - peak[t], max_gain) is
        added to bins k >= 1 before rendering; write_db=True also stores the normalised rows back into `db`, in place.
        Returns dict(points=[S, T, dch, P]) for want_points and pixels=[S, T, dch, P], min=[S, T, 2] for want_pixels."""
        S, T, dch, B = db.shape
        if dch != self.display_channels or B != self.bins:
            raise ValueError(f"db rows are [{dch}][{B}], the engine's are [{self.display_channels}][{self.bins}]")
        if hasattr(db, "data_ptr"):
            import torch
            assert db.is_cuda and db.dtype == torch.float32 and db.is_contiguous()
            mk = lambda shape: torch.empty(shape, dtype=torch.float32, device=db.device)  # noqa: E731
            if stream is None:
                stream = torch.cuda.current_stream(db.device).cuda_stream
            if peak is not None and hasattr(peak, "data_ptr"):
                assert peak.dtype == torch.float32 and peak.is_contiguous()
        else:
            if not (isinstance(db, np.ndarray) and db.dtype == np.float32 and db.flags.c_contiguous):
                if write_db:
                    raise ValueError("write_db needs db as a C-contiguous float32 array (it is updated in place)")
                db = np.ascontiguousarray(db, dtype=np.float32)
            mk = lambda shape: np.empty(shape, dtype=np.float32)  # noqa: E731
        if peak is not None and not hasattr(peak, "data_ptr"):
            peak = np.ascontiguousarray(peak, dtype=np.float32)
        if peak is not None:
            assert tuple(peak.shape) == (T,), peak.shape
        out = {}
        if want_points:
            out["points"] = mk((S, T, dch, self.num_points))
        if want_pixels:
            out["pixels"], out["min"] = mk((S, T, dch, self.num_points)), mk((S, T, 2))
        rb = WfRenderBatch()
        rb.struct_size = C.sizeof(WfRenderBatch)
        rb.n_streams, rb.n_frames = S, T
        rb.db, rb.peak = _ptr(db), _ptr(peak)
        rb.target_db, rb.max_gain, rb.write_db = target_db, max_gain, int(bool(write_db))
        rb.out_points, rb.out_pixels, rb.out_min = _ptr(out.get("points")), _ptr(out.get("pixels")), _ptr(out.get("min"))
        if stream == 0:
            stream = 1  # cudaStreamLegacy; NULL would select the engine's private stream
        self._check(self.L.wf_render(self.h, C.byref(rb), stream))
        return out


def make_meter_config(settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                      device: int = -1, mode: int | None = None) -> WfMeterConfig:
    """Reference setting keys (meter_buf, rms_mode, temporal_smoothing, gravity, fast_peaks, floor, and for the display
    stage height, ceiling, bar_width, rounded_caps, min_bar_height;
    src/settings.hpp:29-135, defaults src/source.cpp:119-174) -> wf_meter_config."""
    L = load_library()
    c = WfMeterConfig()
    L.wf_meter_config_init(C.byref(c))
    s = dict(settings or {})
    c.device, c.max_streams, c.sample_rate = device, max_streams, sample_rate
    c.capture_channels = min(channels, 2)
    c.meter_ms = int(s.pop("meter_buf", 150))
    rms = bool(s.pop("rms_mode", True))
    c.mode = (METER_RMS if rms else METER_PEAK) if mode is None else mode
    c.tsmoothing = TSMOOTH[s.pop("temporal_smoothing", "exp_moving_avg")]
    c.gravity = float(s.pop("gravity", 0.65))
    c.fast_peaks = int(bool(s.pop("fast_peaks", False)))
    c.floor_db = int(s.pop("floor", -65))
    # display stage (render_bars in meter mode)
    c.height = int(s.pop("height", 225))
    c.ceiling_db = int(s.pop("ceiling", 0))
    c.bar_width = int(s.pop("bar_width", 24))
    c.rounded_caps = int(bool(s.pop("rounded_caps", False)))
    c.min_bar_height = int(s.pop("min_bar_height", 0))
    c.sync_offset_ms = int(s.pop("audio_sync_offset", 0))
    if s:
        raise KeyError(f"unsupported meter settings: {sorted(s)}")
    return c


class MeterEngine(_Handle):
    """Level meter (tick_meter) / RMS feed (update_input_rms) on the GPU: ctypes over wf_meter_*; no DSP here."""

    _prefix = "wf_meter"

    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                 device: int = -1, mode: int | None = None):
        self._create(make_meter_config(settings, sample_rate, channels, max_streams, device, mode))
        self.window = int(self.L.wf_meter_window(self.h))

    def reset(self, first_stream=0, count=None):
        count = self.cfg.max_streams - first_stream if count is None else count
        self._check(self.L.wf_meter_reset(self.h, first_stream, count))

    def _state_shapes(self):
        cc, D = self.cfg.capture_channels, _sync_delay(self.cfg.sample_rate, self.cfg.sync_offset_ms)
        parts = {"ring": ((cc, self.window), np.float32), "line": ((cc, D), np.float32), "ema": ((cc,), np.float32),
                 "flags": ((), np.uint8)}
        if self.cfg.mode == METER_INPUT_RMS:
            del parts["ema"]  # the RMS feed has no EMA
        return parts

    def get_state(self, first_stream=0, count=None) -> dict:
        """The state of slots [first_stream, first_stream + count) (wf_meter_get_state): ring [count, cc, window] (the last
        window samples, oldest first), line [count, cc, D] (the sync offset's delay line), ema [count, cc] (m_meter_buf;
        None for INPUT_RMS) and flags [count] (bit0 = m_last_silent)."""
        count = self.cfg.max_streams - first_stream if count is None else count
        st = {k: np.zeros((max(count, 0), *shape), dtype) for k, (shape, dtype) in self._state_shapes().items()}
        self._check(self.L.wf_meter_get_state(self.h, first_stream, count, st["ring"].ctypes.data, st["line"].ctypes.data,
                                              _ptr(st.get("ema")), st["flags"].ctypes.data))
        return {"ring": st["ring"], "line": st["line"], "ema": st.get("ema"), "flags": st["flags"]}

    def set_state(self, state: dict, first_stream=0):
        """Restore slots [first_stream, first_stream + count) from a get_state dict (of this or another engine with the
        same config); a missing or None part is left as it is."""
        count, a = _state_parts(state, self._state_shapes())
        self._check(self.L.wf_meter_set_state(self.h, first_stream, count, _ptr(a["ring"]), _ptr(a["line"]),
                                              _ptr(a.get("ema")), _ptr(a["flags"])))

    def process(self, pcm, n_ticks: int, hop: int, *, first_stream=0, seconds=1.0 / 60.0, stream=None, want_pixels=False,
                pcm_format="f32"):
        """pcm: [n_streams, capture_channels, >= n_ticks*hop] float32, numpy (host) or CUDA torch tensor.
        Returns dict(db, lin, silent) — or dict(rms=[S, T]) for an INPUT_RMS engine.  want_pixels adds the bar heights
        render_bars draws, pixels=[S, T, capture_channels], and min=[S, T, 2] (miny, minpos).  CUDA tensors without an
        explicit `stream` run on torch's current stream.  pcm_format="s16": int16 samples instead (an int16 numpy array or
        a contiguous int16 CUDA tensor), read by the kernels as v * 2**-15; the default converts any numpy array to float32
        as it is, without scaling."""
        fmt = _pcm_format(pcm_format)
        x = _Inputs(pcm, self.cfg.capture_channels, n_ticks * hop, "meter", s16=fmt == PCM_S16)
        S, cc, ns, mk, f32, u8 = x.S, x.cc, x.ns, x.new, x.f32, x.u8
        feed = self.cfg.mode == METER_INPUT_RMS
        out = {"rms": mk((S, n_ticks), f32)} if feed else {
            "db": mk((S, n_ticks, cc), f32), "lin": mk((S, n_ticks, cc), f32), "silent": mk((S, n_ticks), u8)}
        if want_pixels:
            out["pixels"], out["min"] = mk((S, n_ticks, cc), f32), mk((S, n_ticks, 2), f32)
        if stream is None:
            stream = x.stream
        b = WfMeterBatch()
        b.struct_size = C.sizeof(WfMeterBatch)
        b.n_streams, b.n_ticks, b.hop, b.first_stream, b.seconds = S, n_ticks, hop, first_stream, seconds
        b.pcm, b.stream_stride, b.channel_stride = _ptr(x.pcm), cc * ns, ns
        b.out_db = None if feed else _ptr(out["db"])
        b.out_lin = _ptr(out["rms"]) if feed else _ptr(out["lin"])
        b.out_silent = None if feed else _ptr(out["silent"])
        b.out_pixels, b.out_min = _ptr(out.get("pixels")), _ptr(out.get("min"))
        b.pcm_format = fmt
        if stream is None:
            self._check(self.L.wf_meter_process(self.h, C.byref(b)))
        else:
            self._check(self.L.wf_meter_process_async(self.h, C.byref(b), 1 if stream == 0 else stream))
        return out


def make_wave_config(settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                     device: int = -1) -> WfWaveConfig:
    """Reference setting keys (width, meter_buf, channel_mode, normalize_volume, volume_target, max_gain, and for the display
    stage interp_mode, filter_mode, filter_radius, height, floor, ceiling, channel_spacing) -> wf_wave_config."""
    L = load_library()
    c = WfWaveConfig()
    L.wf_wave_config_init(C.byref(c))
    s = dict(settings or {})
    c.device, c.max_streams, c.sample_rate = device, max_streams, sample_rate
    mode = s.pop("channel_mode", "mono")
    c.stereo = int(mode == "stereo")
    c.capture_channels = min(channels, 2) if mode != "single" else 1
    c.width = int(s.pop("width", 800))
    c.meter_ms = int(s.pop("meter_buf", 150))
    c.normalize_volume = int(bool(s.pop("normalize_volume", False)))
    c.volume_target = float(s.pop("volume_target", -8.0))
    c.max_gain = float(s.pop("max_gain", 30.0))
    c.interp_mode = INTERPS[s.pop("interp_mode", "catmull_rom")]
    c.filter_mode = FILTERS[s.pop("filter_mode", "none")]
    c.filter_radius = float(s.pop("filter_radius", 1.5))
    c.height = int(s.pop("height", 225))
    c.floor_db = int(s.pop("floor", -65))
    c.ceiling_db = int(s.pop("ceiling", 0))
    c.channel_spacing = int(s.pop("channel_spacing", 0))
    c.sync_offset_ms = int(s.pop("audio_sync_offset", 0))
    if s:
        raise KeyError(f"unsupported waveform settings: {sorted(s)}")
    return c


class WaveEngine(_Handle):
    """Waveform (oscilloscope) mode (tick_waveform) on the GPU: ctypes over wf_wave_*; no DSP here.  device_clock=True
    keeps the engine's clock and tick plan on the GPU (wf_wave_create_with_clock), so that its calls can be captured into a
    CUDA graph; it is not a plugin setting, and the outputs are the same either way."""

    _prefix = "wf_wave"

    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                 device: int = -1, device_clock: bool = False):
        self.device_clock = bool(device_clock)
        self._create(make_wave_config(settings, sample_rate, channels, max_streams, device), "create_with_clock",
                     int(self.device_clock))
        self.display_channels = 2 if self.cfg.stereo else 1

    def reset(self):
        self._check(self.L.wf_wave_reset(self.h))

    def _state_shapes(self):
        cc, W = self.cfg.capture_channels, self.cfg.width
        och = 2 if (cc > 1 or self.cfg.stereo) else 1  # the m_decibels rows
        D = _sync_delay(self.cfg.sample_rate, self.cfg.sync_offset_ms)
        return {"db": ((och, W), np.float32), "hold": ((cc, D), np.float32), "flags": ((), np.uint8)}

    def get_state(self, first_stream=0, count=None) -> dict:
        """The state of slots [first_stream, first_stream + count) (wf_wave_get_state): db [count, C, width] (m_decibels,
        oldest point first; C = 2 for a stereo capture or stereo display, else 1), hold [count, cc, D] (the sync offset's
        holdback) and flags [count] (bit0 = m_last_silent).  A source's checkpoint also needs the engine's get_clock()."""
        count = self.cfg.max_streams - first_stream if count is None else count
        st = {k: np.zeros((max(count, 0), *shape), dtype) for k, (shape, dtype) in self._state_shapes().items()}
        self._check(self.L.wf_wave_get_state(self.h, first_stream, count, st["db"].ctypes.data, st["hold"].ctypes.data,
                                             st["flags"].ctypes.data))
        return st

    def set_state(self, state: dict, first_stream=0):
        """Restore slots [first_stream, first_stream + count) from a get_state dict; a missing or None part is left as it
        is.  The engine's clock is restored separately (set_clock)."""
        count, a = _state_parts(state, self._state_shapes())
        self._check(self.L.wf_wave_set_state(self.h, first_stream, count, _ptr(a["db"]), _ptr(a["hold"]), _ptr(a["flags"])))

    def get_clock(self) -> dict:
        """The engine-wide clock (wf_wave_get_clock) as dict(clock_ns, audio_ts, waveform_ts, buffered)."""
        c = WfWaveClock()
        self._check(self.L.wf_wave_get_clock(self.h, C.byref(c)))
        return {name: int(getattr(c, name)) for name, _ in WfWaveClock._fields_}

    def set_clock(self, clk):
        """Replace the engine-wide clock with a get_clock() dict, or a (clock_ns, audio_ts, waveform_ts, buffered) tuple,
        of this engine or another with the same config, host or device clock alike.  WfError (WF_ERR_INVALID_ARG) for a
        clock this config's timestamp walk cannot have left; the clock then stays as it was."""
        names = [name for name, _ in WfWaveClock._fields_]
        values = [clk[n] for n in names] if isinstance(clk, dict) else list(clk)
        if len(values) != len(names):
            raise ValueError(f"a clock has {len(names)} fields {names}, got {len(values)}")
        self._check(self.L.wf_wave_set_clock(self.h, C.byref(WfWaveClock(*(int(v) for v in values)))))

    def process(self, pcm, n_ticks: int, hop: int, *, input_rms=None, stream=None, want_db=True, want_points=False,
                want_pixels=False, pcm_format="f32"):
        """pcm: [max_streams, capture_channels, >= n_ticks*hop] float32, numpy (host) or CUDA torch tensor.
        Returns dict(out=[S, T, display_channels, width], silent=[S, T]); want_points / want_pixels add what render_curve
        computes from each tick's rows: points (interpolated + smoothed dB), pixels and min=[S, T, 2] (miny, minpos), all
        [S, T, display_channels, width].  want_db=False leaves `out` out (a display-only call).  CUDA tensors without an
        explicit `stream` run on torch's current stream.  pcm_format="s16": int16 samples instead (an int16 numpy array or
        a contiguous int16 CUDA tensor), read by the kernels as v * 2**-15; the default converts any numpy array to float32
        as it is, without scaling."""
        fmt = _pcm_format(pcm_format)
        x = _Inputs(pcm, self.cfg.capture_channels, n_ticks * hop, s16=fmt == PCM_S16)
        S, cc, ns, mk, f32, u8 = x.S, x.cc, x.ns, x.new, x.f32, x.u8
        input_rms = x.aux(input_rms, f32)
        shape = (S, n_ticks, self.display_channels, self.cfg.width)
        out = {"silent": mk((S, n_ticks), u8)}
        if want_db:
            out["out"] = mk(shape, f32)
        if want_points:
            out["points"] = mk(shape, f32)
        if want_pixels:
            out["pixels"], out["min"] = mk(shape, f32), mk((S, n_ticks, 2), f32)
        if stream is None:
            stream = x.stream
        b = WfWaveBatch()
        b.struct_size = C.sizeof(WfWaveBatch)
        b.n_streams, b.n_ticks, b.hop = S, n_ticks, hop
        b.pcm, b.stream_stride, b.channel_stride = _ptr(x.pcm), cc * ns, ns
        b.input_rms, b.out, b.out_silent = _ptr(input_rms), _ptr(out.get("out")), _ptr(out["silent"])
        b.out_points, b.out_pixels, b.out_min = _ptr(out.get("points")), _ptr(out.get("pixels")), _ptr(out.get("min"))
        b.pcm_format = fmt
        if stream is None:
            self._check(self.L.wf_wave_process(self.h, C.byref(b)))
        else:
            self._check(self.L.wf_wave_process_async(self.h, C.byref(b), 1 if stream == 0 else stream))
        return out


def preview_wave_plan(cfg: WfWaveConfig, n_ticks: int, hop: int):
    """(counts[n_ticks], src[total]) of the first call after wf_wave_create — host arithmetic only, no device."""
    L = load_library()
    counts = np.zeros(n_ticks, np.int32)
    total = L.wf_wave_preview_plan(C.byref(cfg), n_ticks, hop, counts.ctypes.data, None, 0)
    if total < 0:
        raise WfError(int(total), L.wf_strerror(int(total)).decode())
    src = np.zeros(max(int(total), 1), np.int32)
    L.wf_wave_preview_plan(C.byref(cfg), n_ticks, hop, counts.ctypes.data, src.ctypes.data, int(total))
    return counts, src[: int(total)]


def preview_wave_tables(cfg: WfWaveConfig) -> dict:
    """The waveform display stage's tables for a config (wf_wave_preview_table) — host arithmetic only, no device."""
    L = load_library()
    out = {}
    for which, name in ((TABLE_INTERP_INDICES, "interp_indices"), (TABLE_INTERP_WEIGHTS, "interp_weights"),
                        (TABLE_GAUSS, "gauss")):
        n = L.wf_wave_preview_table(C.byref(cfg), which, None, 0)
        if n < 0:
            raise WfError(int(n), L.wf_strerror(int(n)).decode())
        arr = np.zeros(n, dtype=np.float32)
        if n:
            L.wf_wave_preview_table(C.byref(cfg), which, arr.ctypes.data, n)
        out[name] = arr
    return out
