"""B200 linear and salient blending -- drop-in for ``pysteps.blending.linear_blending.forecast``
(pysteps/blending/linear_blending.py).

The host keeps the reference's argument flow: the metadata of ``to_rainrate`` (thresholds, zero
values, Z-R coefficients and their KeyErrors), the 3-D ``precip[-1]`` selection, the squeezes, the
NWP slicing, the member repetition, the shape assertion and the lead loop with its weights.  That
shape logic runs on zero-stride NumPy stand-ins of the fields, so every IndexError, ValueError and
AssertionError the reference raises is raised with its message, before any kernel runs.  The array
arithmetic runs in csrc/blending.cu:
  - the conversion to rain rate (``b200_blend_transform`` / ``b200_blend_unit``);
  - the member repetition as int32 maps from output member to source member (nothing repeated in
    memory), the nan_to_num of the NWP and the NaN fill of the nowcast per output member;
  - the linear blend of every lead in one launch (``b200_blend_linear``);
  - per lead in the blending window the salient blend (``b200_blend_salient``): dense rank of
    ``diff`` over the (n_ens, m, n) slab by a radix sort, then ``_get_ws``.

Deviations: ``10 ** (x / 10)``, ``exp`` and the Box-Cox and Z-R powers are within 16 ulp of NumPy's
(times 2 + |exponent| for Box-Cox with lambda != 0), not bit-identical; the threshold decision of
every pixel is NumPy's (pixels within the bound are recomputed on the host).  A ulp in a converted
value can move a dense rank, so salient output from those transforms is close to, not equal to,
the reference's.  "NQT", fields that are not float32/float64, conversions that change the field's
dtype, shapes the reference only handles by accident (a squeeze that drops a lead or a grid axis)
and slabs of 2^31 values or more raise NotImplementedError.

The nowcast is this package's (``pysteps_b200.nowcasts.get_method``) when it provides the name,
else pysteps' (``pysteps.nowcasts.get_method``: a plug-in or a stock model), whose NumPy result is
uploaded once.  NumPy input returns NumPy; a CUDA-tensor precip returns a CUDA tensor.
"""
import ctypes

import numpy as np
import torch

from .. import _compare, _device, _lib
from ..extrapolation import semilagrangian as _sl
from ..nowcasts import extrapolation as _extrapolation_nowcast
from ..nowcasts import interface as _nowcasts

_FIX_CAP = 1 << 16  # threshold fix-up entries read back without a second transform pass


def forecast(
    precip,
    precip_metadata,
    velocity,
    timesteps,
    timestep,
    nowcast_method,
    precip_nwp=None,
    precip_nwp_metadata=None,
    start_blending=120,
    end_blending=240,
    fill_nwp=True,
    saliency=False,
    nowcast_kwargs=None,
):
    """Same contract as the reference (see its docstring): returns the (timesteps, m, n) or
    (n_ens_members, timesteps, m, n) blended forecast in the NWP field's dtype."""
    if nowcast_kwargs is None:
        nowcast_kwargs = dict()

    if len(precip.shape) == 3:
        precip = precip[-1, :, :]

    timesteps_nowcast = int(end_blending / timestep)

    nowcast_method_func = _nowcast_method(nowcast_method)
    on_device = _device.is_device_tensor(precip)

    if precip_nwp is None:
        now = _call_nowcast(nowcast_method_func, precip, velocity, timesteps, nowcast_kwargs)
        now, _ = to_rainrate(now, precip_metadata)
        return now if on_device else _device.to_host(now)

    now = _call_nowcast(nowcast_method_func, precip, velocity, timesteps_nowcast, nowcast_kwargs)
    now, _ = to_rainrate(now, precip_metadata)
    nwp, _ = to_rainrate(_field(precip_nwp), precip_nwp_metadata)

    plan = _plan(now, nwp, timesteps, timestep, start_blending, end_blending, fill_nwp, saliency)
    out = _blend(now, nwp, plan, fill_nwp)
    return out if on_device else _device.to_host(out)


def _nowcast_method(name):
    try:
        return _nowcasts.get_method(name)
    except (ValueError, TypeError):
        import pysteps.nowcasts.interface as stock
        return stock.get_method(name)


def _call_nowcast(func, precip, velocity, timesteps, kwargs):
    """The nowcast as a device tensor: this package's extrapolation nowcast is called with device
    fields, anything else with the caller's and its result uploaded once."""
    if func is _extrapolation_nowcast.forecast and getattr(precip, "dtype", None) in (
            np.float32, np.float64, torch.float32, torch.float64):
        _device.require_cuda()
        precip = _sl._field_tensor(precip)
    elif _device.is_device_tensor(precip):
        precip = _device.to_host(precip)  # a host nowcast (the Eulerian persistence, pysteps' models)
    return _field(func(precip, velocity, timesteps, **kwargs))


def _field(x):
    if isinstance(x, torch.Tensor) and x.is_cuda:
        t = x.contiguous()
    else:
        _device.require_cuda()
        t = _device.to_device(np.asarray(x) if not isinstance(x, torch.Tensor) else x)
    if t.dtype not in (torch.float32, torch.float64):
        raise NotImplementedError(f"pysteps_b200 blending: fields of dtype {t.dtype} are not supported "
                                  "(float32 or float64)")
    return t


def _np_dtype(t):
    return np.dtype(np.float32) if t.dtype == torch.float32 else np.dtype(np.float64)


def _same_dtype(ex, dt, what):
    if ex.dtype != dt:
        raise NotImplementedError(f"pysteps_b200 blending: {what} changes a {dt} field to {ex.dtype}; "
                                  "not supported")


# ------------------------------------------------------------------------ conversion to rain rate
def to_rainrate(x, metadata, zr_a=None, zr_b=None):
    """utils/conversion.py:to_rainrate on a float32/float64 device tensor: returns a new device
    tensor and the updated metadata."""
    metadata = metadata.copy()
    dt = _np_dtype(x)
    ex = np.zeros(1, dtype=dt)  # the reference's expressions on one value give its result dtypes
    code = _device.dtype_code(x.dtype)

    transform = metadata["transform"]
    kind, lam, thr, zero = 0, 0.0, 0.0, 0.0  # B200_BLEND_COPY
    if transform is not None:
        if transform == "dB":
            thr = metadata.get("threshold", -10.0)
            zero = 0.0
            _same_dtype(10.0 ** (ex / 10.0), dt, "the dB inverse")
            thr = 10.0 ** (thr / 10.0)
            kind = 2
            metadata["transform"] = None
            metadata["threshold"] = thr
            metadata["zerovalue"] = zero
        elif transform in ["BoxCox", "log"]:
            lam = metadata.pop("BoxCox_lambda", 0.0)
            thr = metadata.get("threshold", -10.0)
            zero = 0.0
            if lam == 0.0:
                _same_dtype(np.exp(ex), dt, "the Box-Cox inverse")
                thr = np.exp(thr)
                kind = 3
            else:
                _same_dtype(np.exp(np.log(lam * ex + 1) / lam), dt, "the Box-Cox inverse")
                thr = np.exp(np.log(lam * thr + 1) / lam)
                kind = 4
            metadata["transform"] = None
            metadata["zerovalue"] = zero
            metadata["threshold"] = thr
        elif transform == "NQT":
            raise NotImplementedError("pysteps_b200 blending: the NQT inverse transform is not supported")
        elif transform == "sqrt":
            kind = 1
            metadata["transform"] = None
            metadata["zerovalue"] = metadata["zerovalue"] ** 2
            metadata["threshold"] = metadata["threshold"] ** 2
        else:
            raise ValueError("Unknown transformation %s" % metadata["transform"])

    unit = metadata["unit"]
    unit_args = None
    if unit == "mm/h":
        pass
    elif unit == "mm":
        threshold = metadata["threshold"]
        zerovalue = metadata["zerovalue"]
        acc = float(metadata["accutime"])
        _same_dtype(ex / acc * 60.0, dt, "the mm conversion")
        unit_args = (1, acc, 60.0)
        metadata["threshold"] = threshold / float(metadata["accutime"]) * 60.0
        metadata["zerovalue"] = zerovalue / float(metadata["accutime"]) * 60.0
    elif unit == "dBZ":
        threshold = metadata["threshold"]
        zerovalue = metadata["zerovalue"]
        if zr_a is None:
            zr_a = metadata.get("zr_a", 200.0)
        if zr_b is None:
            zr_b = metadata.get("zr_b", 1.6)
        _same_dtype((ex / zr_a) ** (1.0 / zr_b), dt, "the Z-R conversion")
        if not isinstance(zr_a, (int, float)) or not isinstance(1.0 / zr_b, float):
            raise NotImplementedError("pysteps_b200 blending: Z-R coefficients must be Python numbers")
        unit_args = (2, float(zr_a), 1.0 / zr_b)
        metadata["zr_a"] = zr_a
        metadata["zr_b"] = zr_b
        metadata["threshold"] = (threshold / zr_a) ** (1.0 / zr_b)
        metadata["zerovalue"] = (zerovalue / zr_a) ** (1.0 / zr_b)
    else:
        raise ValueError("Cannot convert unit %s and transform %s to mm/h" % (metadata["unit"], metadata["transform"]))
    metadata["unit"] = "mm/h"

    n = x.numel()
    s = _device.stream_ptr()
    if kind == 0 and unit_args is None:
        return x, metadata  # mm/h untransformed: nothing writes into the field, so no copy
    y = torch.empty_like(x)
    if kind >= 2:
        t_cmp = _compare.comparison_threshold(dt, thr, "blending")[0]
        nfix = torch.zeros(1, dtype=torch.int64, device="cuda")
        cap = min(n, _FIX_CAP)
        while True:
            fix_idx = torch.empty(max(cap, 1), dtype=torch.int64, device="cuda")
            fix_x = torch.empty(max(cap, 1), dtype=torch.float64, device="cuda")
            _lib.call("b200_blend_transform", x.data_ptr(), y.data_ptr(), code, n, kind, float(lam), t_cmp,
                      float(zero), fix_idx.data_ptr(), fix_x.data_ptr(), cap, nfix.data_ptr(), s)
            count = int(nfix.item())  # the one read-back of the conversion
            if count <= cap:
                break
            cap = count
        if count:
            idx = fix_idx[:count]
            xs = _device.to_host(fix_x[:count]).astype(dt)
            with np.errstate(all="ignore"):
                v = _reference_transform(xs, kind, lam)
                v[v < thr] = zero
            vals = _device.to_device(v.astype(np.float64))
            _lib.call("b200_blend_scatter", y.data_ptr(), code, idx.data_ptr(), vals.data_ptr(), count, s)
    elif kind == 1:
        _lib.call("b200_blend_transform", x.data_ptr(), y.data_ptr(), code, n, kind, 0.0, 0.0, 0.0, None, None, 0,
                  None, s)
    if unit_args is not None:
        src = x if kind == 0 else y
        _lib.call("b200_blend_unit", src.data_ptr(), y.data_ptr(), code, n, unit_args[0], unit_args[1],
                  unit_args[2], s)
    return y, metadata


def _reference_transform(R, kind, lam):
    """The reference's inverse transform, in NumPy, for the pixels the device could not decide."""
    if kind == 2:
        return 10.0 ** (R / 10.0)
    if kind == 3:
        return np.exp(R)
    return np.exp(np.log(lam * R + 1) / lam)


# ------------------------------------------------------------------------ shapes, maps and leads
class _Plan:
    pass


def _standin(t):
    return np.broadcast_to(np.zeros((), dtype=_np_dtype(t)), tuple(t.shape))


def _plan(now, nwp, timesteps, timestep, start_blending, end_blending, fill_nwp, saliency):
    """linear_blending.py:140-260 on zero-stride stand-ins: every error of the reference, the member
    maps, and per lead its mode and weights."""
    S_now, S_nwp = _standin(now), _standin(nwp)
    now_members = nwp_members = None  # member axis length of the underlying tensor, or None (3-D)
    if len(S_now.shape) == 4:
        n_now = S_now.shape[0]
        now_members = n_now
        if n_now == 1:
            S_now = np.squeeze(S_now)
    else:
        n_now = 1
    if len(S_nwp.shape) == 4:
        S_nwp = S_nwp[:, 0:timesteps, :, :]
        n_nwp = S_nwp.shape[0]
        nwp_members = n_nwp
        if n_nwp == 1:
            S_nwp = np.squeeze(S_nwp)
    else:
        S_nwp = S_nwp[0:timesteps, :, :]
        n_nwp = 1

    n_max, n_min = max(n_now, n_nwp), min(n_now, n_nwp)
    map_now = np.arange(n_now, dtype=np.int32)
    map_nwp = np.arange(n_nwp, dtype=np.int32)
    if n_min != n_max:
        if n_nwp == 1:
            S_nwp = np.broadcast_to(S_nwp[np.newaxis, :, :], (n_max,) + S_nwp.shape)
            map_nwp = np.zeros(n_max, dtype=np.int32)
        elif n_now == 1:
            S_now = np.broadcast_to(S_now[np.newaxis, :, :], (n_max,) + S_now.shape)
            map_now = np.zeros(n_max, dtype=np.int32)
        else:
            repeats = [(n_max + i) // n_min for i in range(n_min)]
            # consecutive blocks: for 10 and 3 members, 0,0,0,1,1,1,2,2,2,2
            if n_nwp == n_min:
                map_nwp = np.repeat(map_nwp, repeats).astype(np.int32)
                S_nwp = np.broadcast_to(S_nwp[:1], (len(map_nwp),) + S_nwp.shape[1:])
            elif n_now == n_min:
                map_now = np.repeat(map_now, repeats).astype(np.int32)
                S_now = np.broadcast_to(S_now[:1], (len(map_now),) + S_now.shape[1:])

    assert (
        S_nwp.shape[-2:] == S_now.shape[-2:]
    ), "The x and y dimensions of precip_nowcast and precip_nwp need to be identical: dimension of precip_nwp = {} and dimension of precip_nowcast = {}".format(
        S_nwp.shape[-2:], S_now.shape[-2:]
    )

    if fill_nwp:
        src = S_nwp[:, 0:end_lead(end_blending, timestep), :, :] if len(S_nwp.shape) == 4 else \
            S_nwp[0:end_lead(end_blending, timestep), :, :]
        if src.shape != S_now.shape:  # NumPy's IndexError for a mask that does not match; equal shapes cannot fail
            src[np.broadcast_to(np.zeros((), dtype=bool), S_now.shape)]

    S_out = S_nwp
    ref_dim = 0 if n_max == 1 else 1
    plan = _Plan()
    plan.modes, plan.w_nwp, plan.w_now, plan.bits, plan.ws = [], [], [], [], []
    now_dt, nwp_dt = np.zeros((), _np_dtype(now)), np.zeros((), _np_dtype(nwp))
    for i in range(timesteps):
        t = (i + 1) * timestep
        slc = [slice(None)] * S_out.ndim
        slc[ref_dim] = i
        slc = tuple(slc)
        weight_nwp = (t - start_blending) / (end_blending - start_blending)
        if weight_nwp <= 0.0:
            _assign(S_out, slc, S_now[slc])
            plan.modes.append(0)
            plan.w_nwp.append(0.0), plan.w_now.append(0.0), plan.bits.append(0), plan.ws.append(None)
        elif weight_nwp >= 1.0:
            _assign(S_out, slc, S_nwp[slc])
            plan.modes.append(1)
            plan.w_nwp.append(0.0), plan.w_now.append(0.0), plan.bits.append(0), plan.ws.append(None)
        else:
            weight_nowcast = 1.0 - weight_nwp
            if saliency:
                a, b = S_now[slc], S_nwp[slc]
                _broadcast(a, b, "-")
                _broadcast(a, b, "+")
                _assign(S_out, slc, np.broadcast_to(np.zeros((), np.float64), np.broadcast_shapes(a.shape, b.shape)))
                w = weight_nowcast
                try:
                    plan.ws.append((float(w), float(1 - w), float(w**2), float((1 - w) ** 2)))
                except TypeError:
                    raise NotImplementedError("pysteps_b200 blending: weights must be real numbers") from None
                plan.modes.append(3)
                plan.w_nwp.append(0.0), plan.w_now.append(0.0), plan.bits.append(0)
            else:
                b, a = S_nwp[slc], S_now[slc]
                _broadcast(b, a, "+")
                _assign(S_out, slc, np.broadcast_to(np.zeros((), nwp_dt.dtype), np.broadcast_shapes(a.shape, b.shape)))
                pa = (weight_nwp * nwp_dt).dtype
                pb = (weight_nowcast * now_dt).dtype
                ps = np.result_type(np.zeros((), pa), np.zeros((), pb))
                if not all(d in (np.float32, np.float64) for d in (pa, pb, ps)):
                    raise NotImplementedError("pysteps_b200 blending: weights must be real numbers")
                plan.modes.append(2)
                plan.w_nwp.append(float(weight_nwp)), plan.w_now.append(float(weight_nowcast))
                plan.bits.append((pa == np.float64) | (pb == np.float64) << 1 | (ps == np.float64) << 2)
                plan.ws.append(None)

    canonical = (S_now.ndim == S_nwp.ndim == (4 if n_max > 1 else 3) and S_now.shape[-2:] == S_nwp.shape[-2:]
                 and (n_max == 1 or S_now.shape[0] == S_nwp.shape[0] == n_max)
                 and tuple(nwp.shape[-2:]) == S_nwp.shape[-2:] and tuple(now.shape[-2:]) == S_now.shape[-2:]
                 and S_now.ndim - (n_max > 1) == 3)
    if not canonical:
        raise NotImplementedError("pysteps_b200 blending: a squeeze that drops a lead or grid axis is not supported")
    plan.n_out = n_max
    plan.T_out = S_out.shape[ref_dim]
    plan.map_now, plan.map_nwp = map_now, map_nwp  # n_max entries each
    m, n = S_out.shape[-2:]
    plan.P = int(m) * int(n)
    # member strides of the underlying tensors (a 3-D field has one member)
    plan.now_member = int(now.shape[1]) * plan.P if now.ndim == 4 else 0
    plan.nwp_member = int(nwp.shape[1]) * plan.P if nwp.ndim == 4 else 0
    if saliency and plan.n_out * plan.P >= 1 << 31:
        raise NotImplementedError("pysteps_b200 blending: salient slabs of 2^31 values or more are not supported")
    return plan


def end_lead(end_blending, timestep):
    return int(end_blending / timestep)


def _assign(out, slc, value):
    """`out[slc] = value`, with NumPy's errors, without writing into a field"""
    target = out[slc]
    if value.shape != target.shape:
        w = np.lib.stride_tricks.as_strided(np.zeros(1, out.dtype), shape=out.shape, strides=(0,) * out.ndim,
                                            writeable=True)
        w[slc] = value  # raises NumPy's own "could not broadcast ..." when the reference does


def _broadcast(a, b, op):
    try:
        np.broadcast_shapes(a.shape, b.shape)
    except ValueError:
        a + b if op == "+" else a - b  # raises NumPy's own message


def _blend(now, nwp, plan, fill_nwp):
    s = _device.stream_ptr()
    out = torch.empty((plan.n_out, plan.T_out) + tuple(nwp.shape[-2:]), dtype=nwp.dtype, device="cuda")
    d_map_now = _device.to_device(plan.map_now)
    d_map_nwp = _device.to_device(plan.map_nwp)
    d_modes = _device.to_device(np.array(plan.modes, dtype=np.int32))
    d_bits = _device.to_device(np.array(plan.bits, dtype=np.int32))
    d_w = _device.to_device(np.array([plan.w_nwp, plan.w_now], dtype=np.float64).reshape(2, -1))
    args = (now.data_ptr(), _device.dtype_code(now.dtype), d_map_now.data_ptr(), plan.now_member,
            nwp.data_ptr(), _device.dtype_code(nwp.dtype), d_map_nwp.data_ptr(), plan.nwp_member, out.data_ptr(),
            plan.n_out, plan.T_out, plan.P)
    _lib.call("b200_blend_linear", *args, d_modes.data_ptr(), d_bits.data_ptr(), d_w[0].data_ptr(),
              d_w[1].data_ptr(), int(bool(fill_nwp)), s)
    salient = [i for i, md in enumerate(plan.modes) if md == 3]
    if salient:
        nbytes = _lib.c_i64(0)
        _lib.call("b200_blend_scratch_bytes", plan.n_out * plan.P, ctypes.byref(nbytes))
        scratch = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device="cuda")  # reused by every lead
        for i in salient:
            w, w1, w2, w12 = plan.ws[i]
            _lib.call("b200_blend_salient", *args, i, w, w1, w2, w12, int(bool(fill_nwp)), scratch.data_ptr(),
                      nbytes.value, s)
    return out if plan.n_out > 1 else out[0]
