"""One line for the headline grid (config 2 x 32 blocks): device ms and per-kernel ms.  Used for A/B runs of experiment
builds: GB200_LIB=... python tools/quick_grid.py"""
import sys

sys.argv = ["x"]
sys.path.insert(0, "tools")
import bench_configs as b  # noqa: E402

b.grid_case("config 2 x 32 blocks", 2046, 1, 41, 32, 100)
