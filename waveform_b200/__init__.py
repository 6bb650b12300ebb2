"""waveform_b200 — H100 (sm_90a) batched STFT engine behind phandasm/waveform's tick_spectrum seam.

Only what the hot path needs lives here: csrc/ (CUDA kernels + the C-ABI of include/wfstft.h),
host/ (C++ host-side mirror of the plugin's capture/tick plumbing) and this thin ctypes binding.
"""
from .engine import (Engine, MeterEngine, WaveEngine, WfError, load_library, make_config,  # noqa: F401
                     make_meter_config, make_wave_config)
