"""The velocity fix on the CPU: the satellite velocity and clock drift (orbit_core.cuh orbit_velocity, built for the host)
against central differences of the orbit oracle, planted receiver velocities and clock drifts recovered by the host
build of velocity_core.cuh and by the float64 oracle (tests/velocity_oracle.py), the geodetic conversion against the
forward WGS-84 formula, DOP and residuals against numpy, rank deficiency, and the record layout."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import velocity_oracle as vo
from hostbuild import host_library
from velocity_support import (DOP_REL, DRIFT_SS, HEIGHT_M, LAT_DEG, SV_DRIFT_SS, SV_VEL_MS, VEL_MS,
                              velocity_emulator)
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    return velocity_emulator()


def satellite_params(seed, sv):
    """A satellite's world-model parameters after subframes 1-3 of orb.realistic_ephemeris."""
    rng = np.random.default_rng(seed)
    o = orb.OrbitOracle()
    for k, sf in enumerate(orb.ephemeris_subframes(orb.realistic_ephemeris(rng, sv), 3, first_id=1, tow0=20000, seed=seed)):
        o.subframe(orb.parse(orb.words_of(sf)), 1.0 + 6.0 * k)
    return o


def test_satellite_velocity_against_central_difference(emu):
    """orbit_velocity (host build) and the oracle's analytic derivative against (position(t + h) - position(t - h)) / 2h
    with h = 0.1 s, on 16 satellites at times of week around toe and on both sides of both week edges of tk; the clock
    drift against the same difference of the reference's dsv expression."""
    satellite, _, _ = emu
    h = 0.1
    worst = [0.0, 0.0, 0.0]
    for seed in range(16):
        o = satellite_params(seed, 1 + seed)
        p = np.array(o.params()[0])
        toe = p[orb.TOE]
        for dt in (0.0, 1234.5, -5000.25, 302400.0 - 1.0, 302400.0 + 1.0, -302400.0 + 1.0, -302400.0 - 1.0, 7200.0):
            tow = toe + dt
            num = (np.array(o.position(tow + h)) - np.array(o.position(tow - h))) / (2 * h)
            ddsv = (vo.clock_correction(o.p, tow + h) - vo.clock_correction(o.p, tow - h)) / (2 * h)
            got = satellite(p, tow)
            want = np.array(vo.satellite_velocity(o.p, tow))
            worst[0] = max(worst[0], float(np.abs(got[:3] - num).max()), float(np.abs(want[:3] - num).max()))
            worst[1] = max(worst[1], abs(got[3] - ddsv), abs(want[3] - ddsv))
            worst[2] = max(worst[2], float(np.abs(got[:3] - want[:3]).max()))
            assert 2000 < np.linalg.norm(got[:3]) < 5000  # an orbit's speed in the rotating frame
    print(f"worst against the central difference: velocity {worst[0]:.3g} m/s, drift {worst[1]:.3g} s/s; host build "
          f"against the oracle {worst[2]:.3g} m/s")
    assert worst[0] <= SV_VEL_MS and worst[1] <= SV_DRIFT_SS and worst[2] <= 1e-9


def test_clock_drift_keeps_the_reference_af2_square(emu):
    """With af2 set, the drift is af1 + 2 af2^2 (t - toc) + the relativistic rate: the derivative of the reference's
    pow(af2 * (t - toc), 2), not IS-GPS-200's af2 (t - toc)^2."""
    satellite, _, _ = emu
    o = satellite_params(3, 4)
    p = np.array(o.params()[0])
    p[orb.AF2] = 2.0 ** -40
    tow = p[orb.TOC] + 3000.0
    o.p[orb.AF2] = p[orb.AF2]
    base = p.copy()
    base[orb.AF2] = 0.0
    extra = satellite(p, tow)[3] - satellite(base, tow)[3]
    assert extra == pytest.approx(2 * p[orb.AF2] ** 2 * 3000.0, rel=1e-6)
    assert satellite(p, tow)[3] == pytest.approx(vo.satellite_velocity(o.p, tow)[3], rel=1e-12, abs=1e-24)


SITES = [(0.0, 10.0, 0.0), (60.0, -120.0, 9000.0), (89.99, 45.0, -400.0), (-89.99, -170.0, 0.0), (-33.9, 151.2, 9000.0),
         (0.0, 180.0, -400.0), (45.0, 0.0, 0.0)]


def sky(rng, r, n, lat, lon):
    """n satellites 20 200 km up-range from r, above 10 degrees of elevation, with orbital speeds and clock drifts."""
    t = vo.enu_basis(lat, lon)
    out = []
    while len(out) < n:
        az, el = rng.uniform(0, 2 * math.pi), rng.uniform(math.radians(10), math.radians(88))
        d = np.array([math.cos(el) * math.sin(az), math.cos(el) * math.cos(az), math.sin(el)]) @ t
        s = r + 2.02e7 * d
        v = rng.normal(size=3)
        v = 3870.0 * v / np.linalg.norm(v)
        out.append([*s, *v, rng.uniform(-5e-11, 5e-11)])
    return np.array(out)


@pytest.mark.parametrize("n", [4, 5, 8, 12])
def test_planted_velocity_recovered(emu, n):
    """A receiver at each site (equator, 60 N, near both poles; heights -400 m, 0, 9 km) with a planted velocity and
    clock drift; the Dopplers computed exactly from the model.  The host build and the oracle recover the plants."""
    _, compute, _ = emu
    rng = np.random.default_rng(100 + n)
    worst = [0.0, 0.0]
    for lat, lon, h in SITES:
        r = vo.ecef(lat, lon, h)
        sat = sky(rng, r, n, lat, lon)
        v_r = rng.uniform(-300, 300, size=3)
        drift = rng.uniform(-1e-7, 1e-7)
        rows = np.hstack([sat, vo.dopplers(sat, r, v_r, drift)[:, None]])
        for rec in (compute(rows, r), vo.solve(rows, r)):
            assert rec["status"] == vo.VEL_SOLVED and rec["n_rows"] == n
            dv = float(np.abs([rec["vx"] - v_r[0], rec["vy"] - v_r[1], rec["vz"] - v_r[2]]).max())
            dd = abs(rec["clock_drift"] - drift)
            worst = [max(worst[0], dv), max(worst[1], dd)]
            assert dv <= VEL_MS and dd <= DRIFT_SS, (lat, lon, h, dv, dd)
            assert np.isnan(rec["residual_rms"]) == (n == 4)
    print(f"{n} rows: worst velocity {worst[0]:.3g} m/s, drift {worst[1]:.3g} s/s")


def test_geodetic_against_the_forward_formula(emu):
    """Latitudes -90..90 (poles included), longitudes around the globe and heights -10 km .. 100 km: the host build
    returns the point the forward formula started from, within 1e-9 degrees and 1e-4 m, as the oracle does."""
    _, _, geodetic = emu
    rng = np.random.default_rng(7)
    pts = [(lat, lon, h) for lat in (-90.0, -89.999, -60.0, -0.001, 0.0, 30.0, 89.999, 90.0) for lon in (-180.0, -45.0, 0.0, 120.0)
           for h in (-10000.0, -400.0, 0.0, 9000.0, 100000.0)]
    pts += [(rng.uniform(-90, 90), rng.uniform(-180, 180), rng.uniform(-1e4, 1e5)) for _ in range(2000)]
    worst = [0.0, 0.0, 0.0]
    for lat, lon, h in pts:
        x = vo.ecef(lat, lon, h)
        for got in (geodetic(*x), vo.geodetic(*x)):
            dlat = abs(got[0] - lat)
            dlon = abs((got[1] - lon + 180.0) % 360.0 - 180.0) * math.cos(math.radians(lat))  # along the parallel
            dh = abs(got[2] - h)
            worst = [max(worst[0], dlat), max(worst[1], dlon), max(worst[2], dh)]
    print(f"worst latitude {worst[0]:.3g} deg, longitude (scaled to the parallel) {worst[1]:.3g} deg, height {worst[2]:.3g} m")
    assert worst[0] <= LAT_DEG and worst[1] <= LAT_DEG and worst[2] <= HEIGHT_M


def test_geodetic_is_finite_everywhere(emu):
    """The poles (p = 0), the origin, points deep inside the Earth and far outside give finite results; on the axis the
    latitude is +-90 degrees."""
    _, _, geodetic = emu
    for x in [(0.0, 0.0, 0.0), (0.0, 0.0, 6356752.0), (0.0, 0.0, -6356752.0), (0.0, 0.0, 1.0), (1.0, 0.0, 0.0),
              (1e3, -2e3, 5e2), (1e-300, 0.0, 0.0), (1e300, 1e300, -1e300), (4e7, 0.0, 0.0), (0.0, 5e4, 0.0)]:
        g = geodetic(*x)
        assert np.isfinite(g).all(), (x, g)
        assert -90.0 <= g[0] <= 90.0 and -180.0 <= g[1] <= 180.0
    assert geodetic(0.0, 0.0, 6356752.0)[0] == 90.0 and geodetic(0.0, 0.0, -6356752.0)[0] == -90.0
    assert abs(geodetic(0.0, 0.0, 6356752.3142)[2]) < 1e-3


@pytest.mark.parametrize("n", [4, 5, 8, 12])
def test_dop_and_residuals_against_numpy(emu, n):
    """Noisy Dopplers (0.5 Hz): the host build's velocity, drift, DOP and residual RMS against lstsq and inv(G^T G)
    in east/north/up, within 1e-9 relative."""
    _, compute, _ = emu
    rng = np.random.default_rng(200 + n)
    worst = 0.0
    for lat, lon, h in SITES:
        r = vo.ecef(lat, lon, h)
        sat = sky(rng, r, n, lat, lon)
        dop = vo.dopplers(sat, r, rng.uniform(-30, 30, size=3), 1e-8) + rng.normal(scale=0.5, size=n)
        rows = np.hstack([sat, dop[:, None]])
        got, want = compute(rows, r, 1.25), vo.solve(rows, r, 1.25)
        assert got["status"] == want["status"] == vo.VEL_SOLVED and got["receiver_timestamp"] == 1.25
        keys = ["gdop", "pdop", "hdop", "vdop", "tdop"] + (["residual_rms"] if n > 4 else [])
        for k in keys:
            rel = abs(got[k] - want[k]) / abs(want[k])
            worst = max(worst, rel)
            assert rel <= DOP_REL, (k, got[k], want[k])
        assert abs(got["gdop"] ** 2 - got["pdop"] ** 2 - got["tdop"] ** 2) <= 1e-12 * got["gdop"] ** 2
        assert abs(got["pdop"] ** 2 - got["hdop"] ** 2 - got["vdop"] ** 2) <= 1e-12 * got["pdop"] ** 2
        # velocity within the conditioning of the noisy solve
        dv = max(abs(got[k] - want[k]) for k in ("vx", "vy", "vz"))
        assert dv <= 1e-9 * (1 + max(abs(want[k]) for k in ("vx", "vy", "vz"))) * got["gdop"]
    print(f"{n} rows: worst DOP / residual relative difference {worst:.3g}")


def test_rank_deficient_and_non_finite_rows(emu):
    """Two identical rows among four: rank 3, status 2 with NaN velocity and DOP and the geodetic position filled; the
    oracle agrees.  A NaN Doppler gives status 2 too."""
    _, compute, _ = emu
    rng = np.random.default_rng(5)
    r = vo.ecef(52.0, 4.0, 10.0)
    sat = sky(rng, r, 4, 52.0, 4.0)
    sat[3] = sat[1]
    rows = np.hstack([sat, vo.dopplers(sat, r, [1.0, 2.0, 3.0], 0.0)[:, None]])
    for rec in (compute(rows, r), vo.solve(rows, r)):
        assert rec["status"] == vo.VEL_UNSOLVABLE and rec["n_rows"] == 4
        assert all(np.isnan(rec[k]) for k in ("vx", "vy", "vz", "clock_drift", "gdop", "pdop", "hdop", "vdop", "tdop"))
        assert abs(rec["latitude_deg"] - 52.0) < 1e-9 and abs(rec["height"] - 10.0) < 1e-4
    sat = sky(rng, r, 5, 52.0, 4.0)
    rows = np.hstack([sat, vo.dopplers(sat, r, [1.0, 2.0, 3.0], 0.0)[:, None]])
    rows[2, 7] = np.nan
    rec = compute(rows, r)
    assert rec["status"] == vo.VEL_UNSOLVABLE and np.isnan(rec["vx"]) and np.isfinite(rec["height"])


def test_layout_python_c_and_cpp(tmp_path):
    from gypsum_b200._native import VEL_NONE, VEL_SOLVED, VEL_UNSOLVABLE, VELOCITY_DTYPE

    names = list(VELOCITY_DTYPE.names)
    py = [VELOCITY_DTYPE.fields[k][1] for k in names] + [VELOCITY_DTYPE.itemsize]
    assert py == [8 * k for k in range(14)] + [112, 116, 120, 128]
    assert vo.VELOCITY_DTYPE == VELOCITY_DTYPE
    assert (VEL_NONE, VEL_SOLVED, VEL_UNSOLVABLE) == (vo.VEL_NONE, vo.VEL_SOLVED, vo.VEL_UNSOLVABLE) == (0, 1, 2)
    cpp = np.zeros(18, dtype=np.int64)
    host_library("velocity_emu").velocity_emu_layout(cpp.ctypes.data_as(C.c_void_p))
    assert list(cpp) == py
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gypsum_b200.h\"\nint main(void) {\n"
                   + "".join(f'    printf("%d\\n", (int)offsetof(gb200_velocity_fix, {k}));\n' for k in names)
                   + '    printf("%d\\n", (int)sizeof(gb200_velocity_fix));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    c = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert c == py


def test_params_timeline_replays_the_world_model():
    """The GPU tests' per-millisecond parameters: None until a subframe sets a value, then the value it set."""
    o = satellite_params(1, 2)
    words = [orb.words_of(sf) for sf in orb.ephemeris_subframes(orb.realistic_ephemeris(np.random.default_rng(1), 2), 3,
                                                                 first_id=1, tow0=20000, seed=1)]
    chans = [([(nav.KIND_SUBFRAME, w, 1.0 + 6.0 * k, 10 * (k + 1)) for k, w in enumerate(words)], -1)]
    params, _ = vo.params_timeline(chans, 40)
    assert np.isnan(params[0, 9, orb.TOE]) and np.isnan(params[0, 29, orb.I0]) and not np.isnan(params[0, 30]).any()
    assert np.array_equal(params[0, 39, :orb.TOW_LAST], np.array(o.p[:orb.TOW_LAST], dtype=float))
