"""Cases of tests/golden/blending_golden.npz (written by gen_blending_golden.py from the reference's
pysteps.blending.linear_blending.forecast).  build_case(name) -> (args, kwargs) of a forecast call.
EXACT: the cases whose conversions to rain rate are exact, where the device must match bit for bit;
the others ("dB", "dBZ") match within the conversion's bound.  UNSUPPORTED: the reference handles
these only by accident of np.squeeze; the package raises NotImplementedError.  LARGE: cases stored as
seeded pixel samples and a NaN count."""
import numpy as np

MM = {"unit": "mm/h", "transform": None}

# pysteps/tests/test_blending_linear_blending.py's parameter table (the grid is 40 x 40 here)
_TABLE = [
    (5, 30, 60, 20, 45, "eulerian", 1, False, True, False), (5, 30, 60, 20, 45, "eulerian", 2, False, False, False),
    (5, 30, 60, 20, 45, "eulerian", 0, False, False, False), (4, 23, 33, 9, 28, "eulerian", 1, False, False, False),
    (3, 18, 36, 13, 27, "eulerian", 1, False, False, False), (7, 30, 68, 11, 49, "eulerian", 1, False, False, False),
    (7, 30, 68, 11, 49, "eulerian", 1, False, False, True), (10, 100, 160, 25, 130, "eulerian", 1, False, False, False),
    (6, 60, 180, 22, 120, "eulerian", 1, False, False, False), (5, 100, 200, 40, 150, "eulerian", 1, False, False, False),
    (5, 30, 60, 20, 45, "extrapolation", 1, False, False, False), (4, 23, 33, 9, 28, "extrapolation", 1, False, False, False),
    (10, 100, 160, 25, 130, "extrapolation", 1, False, False, False),
    (5, 100, 200, 40, 150, "extrapolation", 1, False, False, True), (5, 30, 60, 20, 45, "eulerian", 1, True, True, False),
    (5, 30, 60, 20, 45, "eulerian", 2, True, False, False), (5, 30, 60, 20, 45, "eulerian", 0, True, False, False),
    (5, 30, 60, 20, 45, "extrapolation", 1, True, False, False), (3, 18, 36, 13, 27, "extrapolation", 1, True, False, False),
]


def _table_case(i):
    timestep, start, end, n_timesteps, _, method, n_models, sal, squeeze, fill = _TABLE[i]
    g = 40
    r_nwp = None
    if n_models:
        r_nwp = np.zeros((n_models, n_timesteps, g, g))
        r_nwp[:, :, : g // 2, :] = 11.0
        if squeeze:
            r_nwp = np.squeeze(r_nwp)
    r_input = np.zeros((4, g, g) if timestep % 2 == 0 else (g, g))
    r_input[..., g // 2:, :] = 11.0
    # transformation.dB_transform(r_input, None, threshold=0.1, zerovalue=-15.0)
    with np.errstate(divide="ignore"):
        r_input = np.where(r_input < 0.1, -15.0, 10.0 * np.log10(np.maximum(r_input, 1e-300)))
    V = np.zeros((2, g, g))
    return ((r_input, {"unit": "mm/h", "transform": "dB"}, V, n_timesteps, timestep, method, r_nwp, dict(MM)),
            dict(start_blending=start, end_blending=end, fill_nwp=fill, saliency=sal))


def _field(rng, shape, dt, special=None):
    R = np.where(rng.random(shape) < 0.4, 0.0, rng.gamma(0.8, 2.0, shape))
    u = rng.random(shape)
    R[u < 0.05] = np.nan
    if special == "inf":
        R[(u > 0.05) & (u < 0.07)] = np.inf
        R[(u > 0.07) & (u < 0.09)] = -np.inf
    return R.astype(dt)


def _case(seed, dt=np.float64, k=3, m=24, n=20, T=8, sal=True, fill=True, special=None, meta=MM, nwp_meta=MM,
          method="eulerian", timestep=10, start=20, end=60, precip=None, nwp=None, P3=False, T_nwp=None):
    rng = np.random.default_rng(seed)
    P = _field(rng, (m, n), dt) if precip is None else precip
    if P3:
        P = np.stack([P * 0.5, P])
    if nwp is None:
        shape = (k, T_nwp or T, m, n) if k > 0 else (T_nwp or T, m, n)
        nwp = _field(rng, shape, dt, special)
    V = rng.uniform(-1, 1, (2, m, n)) if method != "eulerian" else np.zeros((2, m, n))
    return ((P, dict(meta), V, T, timestep, method, nwp, dict(nwp_meta)),
            dict(start_blending=start, end_blending=end, fill_nwp=fill, saliency=sal))


def _special(name):
    rng = np.random.default_rng(99)
    if name == "all_zero":
        return _case(1, precip=np.zeros((24, 20)), nwp=np.zeros((3, 8, 24, 20)))
    if name == "constant_diff":
        return _case(2, precip=np.ones((24, 20)), nwp=np.ones((1, 8, 24, 20)))
    if name == "signed_zero_diff":
        return _case(3, precip=np.zeros((24, 20)), nwp=-np.zeros((3, 8, 24, 20)))
    if name == "nan_diff":  # inf / max = inf / inf: one NaN in diff, scipy's rankdata makes every rank NaN
        P = _field(rng, (24, 20), np.float64)
        P[3, 4] = np.inf
        return _case(4, precip=P)
    raise KeyError(name)


CASES = {}
for _i in range(len(_TABLE)):
    CASES[f"table_{_i}"] = (lambda i=_i: _table_case(i))
for _dt in (np.float32, np.float64):
    for _k in (1, 3, 10, -1):
        for _sal in (False, True):
            for _fill in (False, True):
                _nm = f"{np.dtype(_dt).name}_k{_k}_{'sal' if _sal else 'lin'}_{'fill' if _fill else 'nofill'}"
                CASES[_nm] = (lambda dt=_dt, k=_k, sal=_sal, fill=_fill: _case(
                    7, dt=dt, k=k, m=16, n=12, sal=sal, fill=fill, special="inf"))
for _nm in ("all_zero", "constant_diff", "signed_zero_diff", "nan_diff"):
    CASES[_nm] = (lambda nm=_nm: _special(nm))
CASES.update({
    "nwp_none": lambda: (_case(10)[0][:6] + (None, None), _case(10)[1]),
    "precip_3d": lambda: _case(11, P3=True),
    "T1": lambda: _case(12, T=1, start=0, end=10),
    "T1_fill_mismatch": lambda: _case(12, T=1, start=0, end=20),
    "T1_one_member": lambda: _case(13, k=1, T=1, start=0, end=10),
    "leads_beyond_nowcast": lambda: _case(14, T=12, start=10, end=50),
    "all_before_window": lambda: _case(15, start=200, end=300, T=4, fill=False),
    "all_after_window": lambda: _case(16, start=0, end=5, T=4),
    "extrapolation_f32": lambda: _case(17, dt=np.float32, method="extrapolation"),
    "mm_metadata": lambda: _case(18, meta={"unit": "mm", "transform": None, "accutime": 5, "threshold": 0.1,
                                           "zerovalue": 0.0}),
    "sqrt_metadata": lambda: _case(19, meta={"unit": "mm/h", "transform": "sqrt", "threshold": 0.3, "zerovalue": 0.0}),
    "dbz_metadata": lambda: _case(20, nwp_meta={"unit": "dBZ", "transform": None, "threshold": 0.1, "zerovalue": 0.0}),
    "error_grid_mismatch": lambda: _case(21, nwp=np.zeros((3, 8, 24, 21))),
    "error_missing_accutime": lambda: _case(22, meta={"unit": "mm", "transform": None, "threshold": 0.1,
                                                      "zerovalue": 0.0}),
    "error_unknown_unit": lambda: _case(23, meta={"unit": "inch", "transform": None}),
    "error_short_nwp": lambda: _case(24, nwp=np.ones((3, 2, 24, 20)), T=8),
    "large_512": lambda: _case(25, m=512, n=512, k=3, T=8, dt=np.float32),
})
LARGE = {"large_512"}
UNSUPPORTED = {"T1_one_member"}
EXACT = {c for c in CASES if not c.startswith("table_") and c != "dbz_metadata"}


def build_case(name):
    return CASES[name]()
