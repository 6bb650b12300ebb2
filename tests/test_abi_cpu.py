"""CPU-only checks of the product's C-ABI: the library loads, exports every symbol include/wfstft.h declares,
struct layouts match the header, host-side tables equal the reference's, and without a GPU it FAILS LOUDLY
(no CPU fallback)."""
import ctypes as C
import json
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    from waveform_b200.engine import EXPORTS, load_library

    hdr = (ROOT / "include" / "wfstft.h").read_text()
    declared = sorted(set(re.findall(r"\b(wf_[a-z_0-9]+)\s*\(", hdr)))
    assert declared, "header parse failed"
    L = load_library()
    for name in declared:
        assert hasattr(L, name), f"{name} declared in wfstft.h but not exported"
    assert sorted(EXPORTS) == declared
    assert L.wf_abi_version() == 2


def test_struct_layouts_match_header(tmp_path):
    from waveform_b200.engine import WfBatch, WfConfig, WfInfo

    src = tmp_path / "sz.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(wf_config), sizeof(wf_batch), sizeof(wf_info),'
                   'offsetof(wf_batch,pcm), offsetof(wf_batch,out_peak), offsetof(wf_config,filter_radius));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [C.sizeof(WfConfig), C.sizeof(WfBatch), C.sizeof(WfInfo), WfBatch.pcm.offset,
                                    WfBatch.out_peak.offset, WfConfig.filter_radius.offset]


def test_no_gpu_means_loud_failure_not_fallback():
    import torch
    from waveform_b200 import Engine, WfError

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(WfError) as ei:
        Engine({"fft_size": 2048}, channels=1)
    assert ei.value.status == -4
    assert "no CPU fallback" in str(ei.value)


def test_config_defaults_are_the_plugin_defaults():
    from waveform_b200.engine import WfConfig, load_library

    c = WfConfig()
    load_library().wf_config_init(C.byref(c))
    # src/source.cpp:119-174
    assert (c.fft_size, c.window, c.tsmoothing, c.interp_mode, c.filter_mode) == (4096, 1, 1, 2, 0)
    assert abs(c.gravity - 0.65) < 1e-7 and (c.cutoff_low, c.cutoff_high, c.floor_db, c.ceiling_db) == (30, 17500, -65, 0)
    assert (c.width, c.bar_width, c.bar_gap, c.log_scale) == (800, 24, 6, 1) and c.struct_size == C.sizeof(WfConfig)


def test_unsupported_and_invalid_configs_are_errors():
    from waveform_b200.engine import WfError, make_config, preview_tables

    cfg = make_config({"fft_size": 2048}, channels=3)
    assert cfg.capture_channels == 2                      # the plugin captures at most two (src/source.cpp:1089)
    cfg.capture_channels = 3
    with pytest.raises(WfError) as ei:
        preview_tables(cfg)
    assert ei.value.status == -1
    cfg = make_config({"fft_size": 100}, channels=1)      # clamped like get_settings (src/source.cpp:562-565)
    assert preview_tables(cfg)["info"].fft_size == 128
    cfg = make_config({"fft_size": 2050}, channels=1)
    assert preview_tables(cfg)["info"].fft_size == 2048
    with pytest.raises(KeyError):
        make_config({"render_mode": "solid"})             # display plumbing is outside the hot path


GOLD = sorted((ROOT / "tests" / "golden").glob("case_*.npz"))


@pytest.mark.parametrize("path", GOLD, ids=[p.stem for p in GOLD])
def test_engine_host_tables_equal_reference_tables(path):
    """libwfstft's setup-time tables (wf_tables.cpp) are bit-identical to what WAVSource::update() built."""
    from waveform_b200.engine import make_config, preview_tables

    z = np.load(path, allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    t = preview_tables(make_config(settings, channels=int(z["channels"])))
    for name in ("window", "slope", "rolloff", "interp_indices", "band_widths", "gauss"):
        assert np.array_equal(t[name], z[name].ravel()), name
    assert np.array_equal(t["interp_weights"], z["interp_weights"].ravel())
    assert np.float32(t["info"].window_sum) == z["window_sum"]
    assert np.float32(t["info"].db_min) == z["db_min"]
    assert t["info"].bins == z["db"].shape[-1] and t["info"].num_points == z["points"].shape[-1]


def test_product_never_imports_the_oracle():
    """The product path may not import, link or execute anything under oracle/."""
    for f in list((ROOT / "waveform_b200").rglob("*.py")) + list((ROOT / "waveform_b200").rglob("*.c*")) \
            + list((ROOT / "waveform_b200").rglob("*.h*")) + [ROOT / "include" / "wfstft.h"]:
        txt = f.read_text(errors="ignore")
        assert "oraclebind" not in txt and "refbind" not in txt and "wf_oracle" not in txt and "liboracle" not in txt, f
    out = subprocess.run(["ldd", str(ROOT / "waveform_b200" / "lib" / "libwfstft.so")], capture_output=True, text=True).stdout
    assert "oracle" not in out and "fftw" not in out.lower()


def test_meter_and_wave_struct_layouts_match_header(tmp_path):
    from waveform_b200.engine import WfMeterBatch, WfMeterConfig, WfWaveBatch, WfWaveConfig

    src = tmp_path / "sz2.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(wf_meter_config), sizeof(wf_meter_batch),'
                   'sizeof(wf_wave_config), sizeof(wf_wave_batch), offsetof(wf_meter_batch,pcm), offsetof(wf_meter_batch,out_silent),'
                   'offsetof(wf_wave_batch,pcm), offsetof(wf_wave_batch,out_silent));return 0;}\n')
    exe = tmp_path / "sz2"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [C.sizeof(WfMeterConfig), C.sizeof(WfMeterBatch), C.sizeof(WfWaveConfig),
                                    C.sizeof(WfWaveBatch), WfMeterBatch.pcm.offset, WfMeterBatch.out_silent.offset,
                                    WfWaveBatch.pcm.offset, WfWaveBatch.out_silent.offset]


def test_meter_and_wave_fail_loudly_without_a_gpu_and_reject_bad_configs():
    """wf_meter_create / wf_wave_create: argument errors first (-1 / -7), then WF_ERR_NO_DEVICE (-4) — never a CPU path."""
    import torch
    from waveform_b200 import MeterEngine, WaveEngine, WfError
    from waveform_b200.engine import WfMeterConfig, WfWaveConfig, load_library

    L = load_library()
    h = C.c_void_p()
    mc = WfMeterConfig()
    L.wf_meter_config_init(C.byref(mc))
    mc.capture_channels = 3
    assert L.wf_meter_create(C.byref(mc), C.byref(h)) == -1 and not h.value
    mc.capture_channels = 2
    mc.struct_size = 4
    assert L.wf_meter_create(C.byref(mc), C.byref(h)) == -7
    wc = WfWaveConfig()
    L.wf_wave_config_init(C.byref(wc))
    assert (wc.width, wc.meter_ms, wc.struct_size) == (800, 150, C.sizeof(WfWaveConfig))
    wc.width = 0
    assert L.wf_wave_create(C.byref(wc), C.byref(h)) == -1 and not h.value
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device branch cannot be exercised")
    for ctor in (lambda: MeterEngine({}, channels=2), lambda: WaveEngine({}, channels=2)):
        with pytest.raises(WfError) as ei:
            ctor()
        assert ei.value.status == -4 and "no CPU fallback" in str(ei.value)


def test_hostbind_parses_sysfs(tmp_path):
    """NUMA placement helper used by bench.py's end-to-end leg: sysfs parsing only (no GPU, no affinity change)."""
    from waveform_b200 import hostbind

    assert hostbind.parse_cpulist("0-3,8,10-11\n") == [0, 1, 2, 3, 8, 10, 11]
    assert hostbind.parse_cpulist("") == []
    dev = tmp_path / "bus" / "pci" / "devices" / "0000:1b:00.0"
    dev.mkdir(parents=True)
    (dev / "numa_node").write_text("1\n")
    node = tmp_path / "devices" / "system" / "node" / "node1"
    node.mkdir(parents=True)
    (node / "cpulist").write_text("32-63,96-127\n")
    assert hostbind.numa_node_of_pci("0000:1b:00.0", sysfs=str(tmp_path)) == 1
    assert len(hostbind.cpus_of_node(1, sysfs=str(tmp_path))) == 64
    (dev / "numa_node").write_text("-1\n")
    assert hostbind.numa_node_of_pci("0000:1b:00.0", sysfs=str(tmp_path)) is None
    info = hostbind.bind_to_gpu_node(0, sysfs=str(tmp_path))   # no CUDA device here: reports why, never raises
    assert info["bound"] is False and info["why"]


def test_plugin_binding_compiles_against_the_unmodified_reference():
    """waveform_b200/host/source_cuda.hpp (WAVSourceCUDA) is compiled against the reference's own source.cpp by
    oracle/ref_build (libwaveform_ref_cuda.so).  Without a GPU the engine refuses to start — loudly, through the plugin's
    log — and tick_spectrum() is a no-op: there is no CPU fallback behind the seam either."""
    import torch
    from oracle import refbind

    if not refbind.cuda_seam_available():
        pytest.skip("oracle/_ref/libwaveform_ref_cuda.so not built (needs the reference sources)")
    src = refbind.RefSource({"fft_size": 2048, "window": "hann"}, impl=refbind.IMPL_CUDA, channels=1)
    assert src.fft_size == 2048
    if not torch.cuda.is_available():
        x = (0.1 * np.random.default_rng(0).standard_normal((1, 8192))).astype(np.float32)
        r = src.run_stft(x, 3, 2048)
        assert (r["db"] == src.db_min).all()      # nothing computed: no device, no fallback


def test_zero_weight_taps_equal_the_shortened_kernel_sum():
    """The display stage (csrc/wf_kernels.cuh, kernel_sum) evaluates interpolation points whose window overlaps the spectrum's
    edge with ALL taps — weight 0 and a clamped address for the missing ones — instead of the reference's shortened loop
    (src/filter.hpp:160-169).  The claim that this is the same fp32 sum bit for bit (skipped terms are leading or trailing,
    x*0 = +-0, the sum starts at +0), restated in numpy float32 with the same sequential mul-then-add order."""
    rng = np.random.default_rng(5)
    f32 = np.float32
    for taps in (4, 8):
        radius = taps // 2
        for _ in range(2000):
            sz = int(rng.integers(taps, 64))
            db = (-120.0 * rng.uniform(size=sz)).astype(f32)
            db[rng.uniform(size=sz) < 0.1] = f32(-758.59564)          # DB_MIN entries
            db[rng.uniform(size=sz) < 0.05] = f32(0.0)
            w = rng.normal(size=taps).astype(f32)
            w[rng.uniform(size=taps) < 0.2] = f32(0.0)
            if rng.uniform() < 0.2:
                w = -w
            index = int(rng.integers(0, sz))
            start = index - radius + 1
            stop = min(index + radius + 1, sz)
            ref = f32(0.0)
            for i in range(max(start, 0), stop):                      # the reference's loop
                ref = f32(ref + f32(db[i] * w[i - start]))
            full = f32(0.0)
            for i in range(taps):                                     # all taps, zero weight + clamped address when out of range
                j = start + i
                ok = 0 <= j < sz
                full = f32(full + f32(db[j if ok else 0] * (w[i] if ok else f32(0.0))))
            assert ref.tobytes() == full.tobytes(), (taps, sz, index)
