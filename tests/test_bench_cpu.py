"""CPU: host-side pieces of bench.py that decide what the JSON line says -- the clock sampler's in-region window, the
output dump (--dump-outputs) and the workload description."""
import importlib.util
import os

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)


class _FakeProc:
    def terminate(self):
        pass

    def wait(self, timeout=None):
        return 0

    def kill(self):
        pass

    def poll(self):
        return 0


def _line(mhz, power_cap="Not Active", thermal="Not Active"):
    return "%d, 1965, 900.0, Not Active, %s, Not Active, %s" % (mhz, thermal, power_cap)


def test_clock_sampler_counts_only_the_samples_of_the_timed_region():
    s = bench.ClockSampler(0)
    s.proc = _FakeProc()
    # start-up / warm-up samples (idle clocks, a thermal flag that must NOT leak into the report), then the timed region
    s.lines = [_line(345, thermal="Active"), _line(1965)]
    first = s.mark()
    s.lines += [_line(1700, "Active"), _line(1650, "Active"), _line(1600, "Active")]
    last = s.mark()
    s.lines += [_line(1580, "Active"), _line(300)]  # the sample in flight when the region ended, then idle again
    r = s.stop(first, last)
    assert r["samples"] == 4 and r["sm_mhz"] == 1625.0 and r["sm_max_mhz"] == 1965.0
    assert r["reasons"] == ["sw_power_cap"]


def test_clock_sampler_without_in_region_samples_falls_back_to_the_latest_one():
    s = bench.ClockSampler(0)
    s.proc = _FakeProc()
    s.lines = [_line(1800, "Active")]
    r = s.stop(s.mark(), s.mark())  # a region shorter than the 200 ms sampling period
    assert r["samples"] == 1 and r["sm_mhz"] == 1800.0
    s2 = bench.ClockSampler(0)  # nvidia-smi missing
    assert s2.stop()["sm_mhz"] is None


def test_dump_outputs_is_deterministic_float32_and_bounded(tmp_path):
    import numpy as np
    import torch
    g = torch.Generator().manual_seed(0)
    views = tuple({"pts3d_pred": torch.randn(2, 600, 1000, 3, generator=g), "relative_pose": torch.randn(2, 4, 4, generator=g)}
                  for _ in range(2))
    a = bench.dump_outputs(str(tmp_path / "a"), views)
    b = bench.dump_outputs(str(tmp_path / "b"), views)
    assert a == b and a["view1_pts3d_pred"] == bench.DUMP_SAMPLE and a["view2_relative_pose"] == 32
    total = 0
    for name in a:
        x, y = np.load(tmp_path / "a" / (name + ".npy")), np.load(tmp_path / "b" / (name + ".npy"))
        assert x.dtype == np.float32 and np.array_equal(x, y)
        total += x.nbytes
    assert total <= 64 << 20
    assert np.array_equal(np.load(tmp_path / "a" / "view2_relative_pose.npy"), views[1]["relative_pose"].numpy().reshape(-1))


def test_workload_description_names_the_baseline_config():
    cfg = bench.make_config(16, 2, 384, 512)
    assert "cfg-2" in cfg["workload"] and "512x384" in cfg["workload"]
    assert "model" not in cfg
