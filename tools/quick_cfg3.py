"""One line for config 3 (32x41x10 ms @ 4.092 Msps, one window per call) and the config-5 shape: device ms and per-kernel ms.
A/B aid: GB200_LIB=... python tools/quick_cfg3.py"""
import sys

sys.argv = ["x"]
sys.path.insert(0, "tools")
import bench_configs as b  # noqa: E402

b.grid_case("config 3: 32x41x10 ms @ 4.092 Msps", 4092, 10, 41, 1, 200)
b.grid_case("config 2-like 10 ms @ 2.046 Msps", 2046, 10, 41, 1, 200)
