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
    "wf_get_state", "wf_set_state", "wf_peak_normalize", "wf_launch_count", "wf_last_kernel_ms", "wf_last_kernel_name",
    "wf_host_alloc", "wf_host_free", "wf_preview_table",
    "wf_meter_config_init", "wf_meter_create", "wf_meter_destroy", "wf_meter_last_error", "wf_meter_window",
    "wf_meter_process", "wf_meter_process_async", "wf_meter_reset", "wf_meter_launch_count", "wf_meter_last_kernel_ms",
    "wf_wave_config_init", "wf_wave_create", "wf_wave_destroy", "wf_wave_last_error", "wf_wave_process",
    "wf_wave_process_async", "wf_wave_reset", "wf_wave_launch_count", "wf_wave_last_kernel_ms", "wf_wave_preview_plan",
]

METER_PEAK, METER_RMS, METER_INPUT_RMS = 0, 1, 2


class WfMeterConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_streams", C.c_int32), ("sample_rate", C.c_uint32),
        ("capture_channels", C.c_int32), ("mode", C.c_int32), ("meter_ms", C.c_int32), ("tsmoothing", C.c_int32),
        ("gravity", C.c_float), ("fast_peaks", C.c_int32), ("floor_db", C.c_int32),
    ]


class WfWaveConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_streams", C.c_int32), ("sample_rate", C.c_uint32),
        ("capture_channels", C.c_int32), ("stereo", C.c_int32), ("width", C.c_int32), ("meter_ms", C.c_int32),
        ("normalize_volume", C.c_int32), ("volume_target", C.c_float), ("max_gain", C.c_float),
    ]


class WfWaveBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_ticks", C.c_int32), ("hop", C.c_int32),
        ("pcm", C.c_void_p), ("stream_stride", C.c_int64), ("channel_stride", C.c_int64),
        ("input_rms", C.c_void_p), ("out", C.c_void_p), ("out_silent", C.c_void_p),
    ]


class WfMeterBatch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("n_streams", C.c_int32), ("n_ticks", C.c_int32), ("hop", C.c_int32),
        ("first_stream", C.c_int32), ("seconds", C.c_float),
        ("pcm", C.c_void_p), ("stream_stride", C.c_int64), ("channel_stride", C.c_int64),
        ("out_db", C.c_void_p), ("out_lin", C.c_void_p), ("out_silent", C.c_void_p),
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
    L.wf_peak_normalize.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_float, C.c_float, vp]
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
    L.wf_meter_launch_count.restype = C.c_int64
    L.wf_meter_launch_count.argtypes = [vp]
    L.wf_meter_last_kernel_ms.restype = C.c_float
    L.wf_meter_last_kernel_ms.argtypes = [vp]
    L.wf_wave_config_init.argtypes = [C.POINTER(WfWaveConfig)]
    L.wf_wave_create.argtypes = [C.POINTER(WfWaveConfig), C.POINTER(vp)]
    L.wf_wave_destroy.argtypes = [vp]
    L.wf_wave_last_error.restype = C.c_char_p
    L.wf_wave_last_error.argtypes = [vp]
    L.wf_wave_process.argtypes = [vp, C.POINTER(WfWaveBatch)]
    L.wf_wave_process_async.argtypes = [vp, C.POINTER(WfWaveBatch), vp]
    L.wf_wave_reset.argtypes = [vp]
    L.wf_wave_launch_count.restype = C.c_int64
    L.wf_wave_launch_count.argtypes = [vp]
    L.wf_wave_last_kernel_ms.restype = C.c_float
    L.wf_wave_last_kernel_ms.argtypes = [vp]
    L.wf_wave_preview_plan.restype = C.c_int64
    L.wf_wave_preview_plan.argtypes = [C.POINTER(WfWaveConfig), C.c_int32, C.c_int32, vp, vp, C.c_int64]
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
        "min_bar_height": "min_bar_height",
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
        elif k in ("auto_fft_size", "audio_sync_offset"):
            pass  # display / capture plumbing that stays on the host side of the seam
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


class Engine:
    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2,
                 max_streams: int = 1, device: int = -1, config: WfConfig | None = None):
        self.L = load_library()
        self.cfg = config if config is not None else make_config(settings, sample_rate, channels, max_streams, device)
        h = C.c_void_p()
        rc = self.L.wf_create(C.byref(self.cfg), C.byref(h))
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_last_error(None).decode()}")
        self.h = h
        self.info = WfInfo()
        self._check(self.L.wf_get_info(self.h, C.byref(self.info)))

    # ---- plumbing ----
    def _check(self, rc):
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.L.wf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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

    @property
    def launch_count(self) -> int:
        return int(self.L.wf_launch_count(self.h))

    def last_kernel_ms(self) -> float:
        return float(self.L.wf_last_kernel_ms(self.h))

    def last_kernel_name(self) -> str:
        return self.L.wf_last_kernel_name(self.h).decode()

    # ---- processing ----
    def process_raw(self, pcm_ptr, n_streams, n_frames, hop, stream_stride, channel_stride, *, first_stream=0,
                    seconds=1.0 / 60.0, input_rms=None, skip_mask=None, out_db=None, out_points=None,
                    out_silent=None, out_peak=None, out_pixels=None, out_min=None, stream=None, sync=True,
                    frame_seconds=None):
        """Thin wrapper over wf_process / wf_process_async with raw pointers (ints)."""
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
        if sync and stream is None:
            self._check(self.L.wf_process(self.h, C.byref(b)))
        else:
            if stream == 0:
                stream = 1  # the legacy default stream is cudaStreamLegacy (0x1); NULL selects the engine's own stream
            self._check(self.L.wf_process_async(self.h, C.byref(b), stream))

    def process(self, pcm, n_frames: int, hop: int, *, first_stream=0, seconds=1.0 / 60.0, input_rms=None,
                skip_mask=None, want_db=True, want_points=False, want_silent=True, want_peak=False, want_pixels=False,
                frame_seconds=None):
        """pcm: [n_streams, capture_channels, samples] float32 — numpy (host path, staged inside the C call)
        or a CUDA torch tensor (device path, outputs are CUDA tensors)."""
        is_torch = hasattr(pcm, "data_ptr")
        if pcm.ndim == 2:
            pcm = pcm[None]
        S, cc, ns = pcm.shape
        if cc != self.capture_channels:
            raise ValueError(f"pcm has {cc} channels, engine captures {self.capture_channels}")
        need = (n_frames - 1) * hop + self.fft_size
        if ns < need:
            raise ValueError(f"need {need} samples per channel, got {ns}")
        dch, B, P = self.display_channels, self.bins, self.num_points
        out = {}
        if is_torch:
            import torch
            assert pcm.is_cuda and pcm.dtype == torch.float32 and pcm.is_contiguous()
            mk = lambda shape, dt: torch.empty(shape, dtype=dt, device=pcm.device)
            f32, u8 = torch.float32, torch.uint8
            if input_rms is not None:
                input_rms = input_rms.to(device=pcm.device, dtype=f32).contiguous()
            if skip_mask is not None:
                skip_mask = skip_mask.to(device=pcm.device, dtype=u8).contiguous()
        else:
            pcm = np.ascontiguousarray(pcm, dtype=np.float32)
            mk = lambda shape, dt: np.empty(shape, dtype=dt)
            f32, u8 = np.float32, np.uint8
            if input_rms is not None:
                input_rms = np.ascontiguousarray(input_rms, dtype=np.float32)
            if skip_mask is not None:
                skip_mask = np.ascontiguousarray(skip_mask, dtype=np.uint8)
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
        stream = None
        if is_torch:
            import torch
            stream = torch.cuda.current_stream(pcm.device).cuda_stream
        fs = None
        if frame_seconds is not None:  # per-tick `seconds` (always a host array), see wf_batch.frame_seconds
            fs = np.ascontiguousarray(frame_seconds, dtype=np.float32)
            assert fs.shape == (n_frames,)
        self.process_raw(_ptr(pcm), S, n_frames, hop, cc * ns, ns, first_stream=first_stream, seconds=seconds,
                         input_rms=_ptr(input_rms), skip_mask=_ptr(skip_mask), out_db=_ptr(out.get("db")),
                         out_points=_ptr(out.get("points")), out_silent=_ptr(out.get("silent")),
                         out_peak=_ptr(out.get("peak")), out_pixels=_ptr(out.get("pixels")), out_min=_ptr(out.get("min")),
                         stream=stream, sync=not is_torch, frame_seconds=None if fs is None else fs.ctypes.data)
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


def make_meter_config(settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                      device: int = -1, mode: int | None = None) -> WfMeterConfig:
    """Reference setting keys (meter_buf, rms_mode, temporal_smoothing, gravity, fast_peaks, floor;
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
    if s:
        raise KeyError(f"unsupported meter settings: {sorted(s)}")
    return c


class MeterEngine:
    """Level meter (tick_meter) / RMS feed (update_input_rms) on the GPU: ctypes over wf_meter_*; no DSP here."""

    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                 device: int = -1, mode: int | None = None):
        self.L = load_library()
        self.cfg = make_meter_config(settings, sample_rate, channels, max_streams, device, mode)
        h = C.c_void_p()
        rc = self.L.wf_meter_create(C.byref(self.cfg), C.byref(h))
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_meter_last_error(None).decode()}")
        self.h = h
        self.window = int(self.L.wf_meter_window(self.h))

    def _check(self, rc):
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_meter_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.L.wf_meter_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return int(self.L.wf_meter_launch_count(self.h))

    def last_kernel_ms(self) -> float:
        return float(self.L.wf_meter_last_kernel_ms(self.h))

    def reset(self, first_stream=0, count=None):
        count = self.cfg.max_streams - first_stream if count is None else count
        self._check(self.L.wf_meter_reset(self.h, first_stream, count))

    def process(self, pcm, n_ticks: int, hop: int, *, first_stream=0, seconds=1.0 / 60.0, stream=None):
        """pcm: [n_streams, capture_channels, >= n_ticks*hop] float32, numpy (host) or CUDA torch tensor.
        Returns dict(db, lin, silent) — or dict(rms=[S, T]) for an INPUT_RMS engine."""
        is_torch = hasattr(pcm, "data_ptr")
        if pcm.ndim == 2:
            pcm = pcm[None]
        S, cc, ns = pcm.shape
        if cc != self.cfg.capture_channels:
            raise ValueError(f"pcm has {cc} channels, meter captures {self.cfg.capture_channels}")
        if ns < n_ticks * hop:
            raise ValueError(f"need {n_ticks * hop} samples per channel, got {ns}")
        if is_torch:
            import torch
            assert pcm.is_cuda and pcm.dtype == torch.float32 and pcm.is_contiguous()
            mk = lambda shape, dt: torch.empty(shape, dtype=dt, device=pcm.device)
            f32, u8 = torch.float32, torch.uint8
        else:
            pcm = np.ascontiguousarray(pcm, dtype=np.float32)
            mk = lambda shape, dt: np.empty(shape, dtype=dt)
            f32, u8 = np.float32, np.uint8
        feed = self.cfg.mode == METER_INPUT_RMS
        out = {"rms": mk((S, n_ticks), f32)} if feed else {
            "db": mk((S, n_ticks, cc), f32), "lin": mk((S, n_ticks, cc), f32), "silent": mk((S, n_ticks), u8)}
        b = WfMeterBatch()
        b.struct_size = C.sizeof(WfMeterBatch)
        b.n_streams, b.n_ticks, b.hop, b.first_stream, b.seconds = S, n_ticks, hop, first_stream, seconds
        b.pcm, b.stream_stride, b.channel_stride = _ptr(pcm), cc * ns, ns
        b.out_db = None if feed else _ptr(out["db"])
        b.out_lin = _ptr(out["rms"]) if feed else _ptr(out["lin"])
        b.out_silent = None if feed else _ptr(out["silent"])
        if stream is None:
            self._check(self.L.wf_meter_process(self.h, C.byref(b)))
        else:
            self._check(self.L.wf_meter_process_async(self.h, C.byref(b), 1 if stream == 0 else stream))
        return out


def make_wave_config(settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                     device: int = -1) -> WfWaveConfig:
    """Reference setting keys (width, meter_buf, channel_mode, normalize_volume, volume_target, max_gain) -> wf_wave_config."""
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
    if s:
        raise KeyError(f"unsupported waveform settings: {sorted(s)}")
    return c


class WaveEngine:
    """Waveform (oscilloscope) mode (tick_waveform) on the GPU: ctypes over wf_wave_*; no DSP here."""

    def __init__(self, settings: dict | None = None, sample_rate: int = 48000, channels: int = 2, max_streams: int = 1,
                 device: int = -1):
        self.L = load_library()
        self.cfg = make_wave_config(settings, sample_rate, channels, max_streams, device)
        h = C.c_void_p()
        rc = self.L.wf_wave_create(C.byref(self.cfg), C.byref(h))
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_wave_last_error(None).decode()}")
        self.h = h
        self.display_channels = 2 if self.cfg.stereo else 1

    def _check(self, rc):
        if rc != WF_OK:
            raise WfError(rc, f"{self.L.wf_strerror(rc).decode()}: {self.L.wf_wave_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.L.wf_wave_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return int(self.L.wf_wave_launch_count(self.h))

    def last_kernel_ms(self) -> float:
        return float(self.L.wf_wave_last_kernel_ms(self.h))

    def reset(self):
        self._check(self.L.wf_wave_reset(self.h))

    def process(self, pcm, n_ticks: int, hop: int, *, input_rms=None, stream=None):
        """pcm: [max_streams, capture_channels, >= n_ticks*hop] float32, numpy (host) or CUDA torch tensor.
        Returns dict(out=[S, T, display_channels, width], silent=[S, T])."""
        is_torch = hasattr(pcm, "data_ptr")
        if pcm.ndim == 2:
            pcm = pcm[None]
        S, cc, ns = pcm.shape
        if cc != self.cfg.capture_channels:
            raise ValueError(f"pcm has {cc} channels, engine captures {self.cfg.capture_channels}")
        if ns < n_ticks * hop:
            raise ValueError(f"need {n_ticks * hop} samples per channel, got {ns}")
        if is_torch:
            import torch
            assert pcm.is_cuda and pcm.dtype == torch.float32 and pcm.is_contiguous()
            mk = lambda shape, dt: torch.empty(shape, dtype=dt, device=pcm.device)
            f32, u8 = torch.float32, torch.uint8
            if input_rms is not None:
                input_rms = input_rms.to(device=pcm.device, dtype=f32).contiguous()
        else:
            pcm = np.ascontiguousarray(pcm, dtype=np.float32)
            mk = lambda shape, dt: np.empty(shape, dtype=dt)
            f32, u8 = np.float32, np.uint8
            if input_rms is not None:
                input_rms = np.ascontiguousarray(input_rms, dtype=np.float32)
        out = {"out": mk((S, n_ticks, self.display_channels, self.cfg.width), f32), "silent": mk((S, n_ticks), u8)}
        b = WfWaveBatch()
        b.struct_size = C.sizeof(WfWaveBatch)
        b.n_streams, b.n_ticks, b.hop = S, n_ticks, hop
        b.pcm, b.stream_stride, b.channel_stride = _ptr(pcm), cc * ns, ns
        b.input_rms, b.out, b.out_silent = _ptr(input_rms), _ptr(out["out"]), _ptr(out["silent"])
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
