"""A float64 oracle of the velocity fix (gypsum_b200/csrc/velocity_core.cuh, DESIGN.md §8d): the satellite's velocity
and clock drift as the analytic derivative of oracle/orbit_oracle.py's position and clock correction, the receiver's
velocity and drift by np.linalg.lstsq, DOP by np.linalg.inv, and the WGS-84 geodetic position iterated to convergence.
Independent of the device code: numpy and math only."""
import math

import numpy as np

from oracle import orbit_oracle as orb

C_LIGHT = 2.99792458e8
L1_HZ = 1575.42e6
WE = 7.2921151467e-5
F_REL = -4.442807633e-10
WGS84_A = 6378137.0
WGS84_F = 1.0 / 298.257223563
WGS84_E2 = WGS84_F * (2.0 - WGS84_F)

VELOCITY_DTYPE = np.dtype([  # gb200_velocity_fix
    ("receiver_timestamp", "<f8"), ("vx", "<f8"), ("vy", "<f8"), ("vz", "<f8"), ("clock_drift", "<f8"),
    ("latitude_deg", "<f8"), ("longitude_deg", "<f8"), ("height", "<f8"), ("gdop", "<f8"), ("pdop", "<f8"),
    ("hdop", "<f8"), ("vdop", "<f8"), ("tdop", "<f8"), ("residual_rms", "<f8"), ("status", "<i4"), ("n_rows", "<i4"),
    ("reserved", "<i4", (2,))])
VEL_NONE, VEL_SOLVED, VEL_UNSOLVABLE = 0, 1, 2


def satellite_velocity(p, tow):
    """(vx, vy, vz, drift) of a satellite with world-model parameters p (OrbitOracle.p order) at time of week tow: the
    time derivative of OrbitOracle.position in its frame and of the clock correction (clock_correction), with t = tow."""
    p = [float(v) for v in p]
    tk = tow - p[orb.TOE]
    if tk > 302_400:
        tk -= 604_800
    elif tk < -302_400:
        tk += 604_800
    e = p[orb.E]
    n = math.sqrt(3.986004418e14) / math.sqrt(math.pow(math.pow(p[orb.SQRT_A], 2), 3)) + p[orb.DN]
    m = p[orb.M0] + n * tk
    ek = m
    for _ in range(7):
        ek = m + e * math.sin(ek)
    ekd = n / (1 - e * math.cos(ek))
    vk = math.atan2(math.sqrt(1 - e * e) * math.sin(ek), math.cos(ek) - e)
    vkd = math.sqrt(1 - e * e) * ekd / (1 - e * math.cos(ek))
    phi = vk + p[orb.OMEGA]
    s2, c2 = math.sin(2 * phi), math.cos(2 * phi)
    uk = phi + p[orb.CUS] * s2 + p[orb.CUC] * c2
    ukd = vkd * (1 + 2 * (p[orb.CUS] * c2 - p[orb.CUC] * s2))
    rk = p[orb.A] * (1 - e * math.cos(ek)) + p[orb.CRS] * s2 + p[orb.CRC] * c2
    rkd = p[orb.A] * e * math.sin(ek) * ekd + 2 * vkd * (p[orb.CRS] * c2 - p[orb.CRC] * s2)
    ik = p[orb.I0] + p[orb.IDOT] * tk + p[orb.CIS] * s2 + p[orb.CIC] * c2
    ikd = p[orb.IDOT] + 2 * vkd * (p[orb.CIS] * c2 - p[orb.CIC] * s2)
    xp, yp = rk * math.cos(uk), rk * math.sin(uk)
    xpd = rkd * math.cos(uk) - rk * ukd * math.sin(uk)
    ypd = rkd * math.sin(uk) + rk * ukd * math.cos(uk)
    omd = p[orb.OMEGA_DOT] - WE
    om = p[orb.OMEGA0] + omd * tk - WE * p[orb.TOE]
    # d/dt of R3(-om) R1(-ik) (xp, yp, 0)
    dx = np.array([xpd, ypd * math.cos(ik) - yp * math.sin(ik) * ikd, ypd * math.sin(ik) + yp * math.cos(ik) * ikd])
    pos = np.array([xp, yp * math.cos(ik), yp * math.sin(ik)])
    co, so = math.cos(om), math.sin(om)
    rot = np.array([[co, -so, 0.0], [so, co, 0.0], [0.0, 0.0, 1.0]])
    drot = omd * np.array([[-so, -co, 0.0], [co, -so, 0.0], [0.0, 0.0, 0.0]])
    v = rot @ dx + drot @ pos
    # the reference's dsv takes Ek at tow - toe without the week wrap
    m = p[orb.M0] + n * (tow - p[orb.TOE])
    ec = m
    for _ in range(7):
        ec = m + e * math.sin(ec)
    drift = (p[orb.AF1] + 2 * p[orb.AF2] ** 2 * (tow - p[orb.TOC])
             + F_REL * e * p[orb.SQRT_A] * math.cos(ec) * n / (1 - e * math.cos(ec)))
    return float(v[0]), float(v[1]), float(v[2]), drift


def clock_correction(p, t):
    """The reference's dsv expression (world_model.py:686) at time t with Ek at t - toe (no iteration on dsv)."""
    p = [float(v) for v in p]
    o = orb.OrbitOracle()
    o.p = list(p)
    ek = o._ecc(t - p[orb.TOE])
    return (p[orb.AF0] + p[orb.AF1] * (t - p[orb.TOC]) + math.pow(p[orb.AF2] * (t - p[orb.TOC]), 2)
            + F_REL * p[orb.E] * p[orb.SQRT_A] * math.sin(ek) - p[orb.TGD])


def geodetic(x, y, z):
    """WGS-84 (latitude deg, longitude deg, height m), latitude iterated until it stops changing."""
    p = math.hypot(x, y)
    lat = math.atan2(z, p * (1 - WGS84_E2))
    for _ in range(100):
        n = WGS84_A / math.sqrt(1 - WGS84_E2 * math.sin(lat) ** 2)
        new = math.atan2(z + WGS84_E2 * n * math.sin(lat), p)
        if new == lat:
            break
        lat = new
    n = WGS84_A / math.sqrt(1 - WGS84_E2 * math.sin(lat) ** 2)
    h = p * math.cos(lat) + z * math.sin(lat) - WGS84_A ** 2 / n
    return math.degrees(lat), math.degrees(math.atan2(y, x)), h


def ecef(lat_deg, lon_deg, h):
    """The forward WGS-84 formula."""
    lat, lon = math.radians(lat_deg), math.radians(lon_deg)
    n = WGS84_A / math.sqrt(1 - WGS84_E2 * math.sin(lat) ** 2)
    return np.array([(n + h) * math.cos(lat) * math.cos(lon), (n + h) * math.cos(lat) * math.sin(lon),
                     (n * (1 - WGS84_E2) + h) * math.sin(lat)])


def enu_basis(lat_deg, lon_deg):
    """Rows east, north, up at a geodetic position."""
    lat, lon = math.radians(lat_deg), math.radians(lon_deg)
    sl, cl, sp, cp = math.sin(lon), math.cos(lon), math.sin(lat), math.cos(lat)
    return np.array([[-sl, cl, 0.0], [-sp * cl, -sp * sl, cp], [cp * cl, cp * sl, sp]])


def solve(rows, r, receiver_timestamp=0.0):
    """The record of one millisecond with a solved fix at r from rows [n][8] of (satellite x, y, z, vx, vy, vz, clock
    drift, Doppler Hz)."""
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 8)
    r = np.asarray(r, dtype=np.float64)
    out = np.zeros(1, dtype=VELOCITY_DTYPE)[0]
    for k in VELOCITY_DTYPE.names[:14]:
        out[k] = np.nan
    out["receiver_timestamp"] = receiver_timestamp
    out["latitude_deg"], out["longitude_deg"], out["height"] = geodetic(*r)
    out["n_rows"] = len(rows)
    out["status"] = VEL_UNSOLVABLE
    d = rows[:, :3] - r
    u = d / np.linalg.norm(d, axis=1)[:, None]
    g = np.hstack([-u, np.ones((len(rows), 1))])
    b = -(C_LIGHT / L1_HZ) * rows[:, 7] - np.sum(u * rows[:, 3:6], axis=1) + C_LIGHT * rows[:, 6]
    if len(rows) < 4 or not np.isfinite(g).all() or not np.isfinite(b).all():
        return out
    x, _, rank, _ = np.linalg.lstsq(g, b, rcond=None)
    if rank < 4:
        return out
    out["vx"], out["vy"], out["vz"] = x[:3]
    out["clock_drift"] = x[3] / C_LIGHT
    if len(rows) > 4:
        out["residual_rms"] = math.sqrt(float(np.mean((b - g @ x) ** 2)))
    q = np.linalg.inv(g.T @ g)
    t = enu_basis(out["latitude_deg"], out["longitude_deg"])
    qenu = t @ q[:3, :3] @ t.T
    out["pdop"] = math.sqrt(np.trace(q[:3, :3]))
    out["tdop"] = math.sqrt(q[3, 3])
    out["gdop"] = math.sqrt(np.trace(q))
    out["hdop"] = math.sqrt(qenu[0, 0] + qenu[1, 1])
    out["vdop"] = math.sqrt(qenu[2, 2])
    out["status"] = VEL_SOLVED
    return out


def dopplers(sat, r, v_r, drift_r):
    """The Dopplers (Hz) that receiver velocity v_r and clock drift drift_r at r measure from satellites sat [n][7] of
    (x, y, z, vx, vy, vz, drift): the model of solve, exactly."""
    sat = np.asarray(sat, dtype=np.float64)
    d = sat[:, :3] - np.asarray(r)
    u = d / np.linalg.norm(d, axis=1)[:, None]
    rate = np.sum(u * (sat[:, 3:6] - np.asarray(v_r)), axis=1) + C_LIGHT * (drift_r - sat[:, 6])
    return -rate * (L1_HZ / C_LIGHT)


def params_timeline(chans, n_ms, sv=None):
    """Every channel's world-model parameters (float64 [n_ms][26], NaN where None) at the end of every millisecond of
    one call, chans [(events [(kind, words, trailing_edge, ms)], drop_ms)], replayed through oracle/orbit_oracle.py.  sv:
    the channels' OrbitOracle entries carried from the call before (None: fresh).  Returns (params, sv)."""
    sv = sv if sv is not None else [orb.OrbitOracle() for _ in chans]
    out = np.full((len(chans), n_ms, orb.N_PARAMS), np.nan)
    for c, (events, drop) in enumerate(chans):
        _replay(sv[c], events, drop, n_ms, out[c])
    return out, sv


def _replay(o, events, drop_ms, n_ms, out):
    """orb.run_call, keeping the parameters after every millisecond in out [n_ms][26]."""
    by_ms: dict = {}
    for kind, w, te, ms in events:
        by_ms.setdefault(ms, []).append((kind, w, te))
    tracked = True
    for m in range(n_ms):
        tracked = orb.step(o, by_ms.get(m, []), m == drop_ms, tracked)
        out[m] = [np.nan if v is None else float(v) for v in o.p]
