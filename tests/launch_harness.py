"""What the per-launch tests share: sentinel-guarded outputs, offset pointers, split fp16 operands, launch signatures, a recorder of C calls,
the plan assertions, and an r3dp_mf_conv3d launch from a plan row.  It imports only torch and ctypes, and the package's C API inside the
helpers that call it, so the CPU-only reference modules (and the fixture generators, which put only tests/ on sys.path) can import it."""
import ctypes

import torch

F16 = torch.float16
#: dtype -> (integer view, bit pattern) of the sentinel a guarded buffer holds: NaN payloads no kernel writes (fp16, fp32, fp64), 0xA5
#: for the uint8 frames and scratch, and an int64 no kernel writes
SENTINEL = {F16: (torch.int16, 0x7E55), torch.float32: (torch.int32, 0x7FC01234), torch.float64: (torch.int64, 0x7FF8000012345678),
            torch.uint8: (torch.uint8, 0xA5), torch.int64: (torch.int64, 0x5A5A5A5A5A5A5A5A)}
GUARD = 4096


# ---- guarded outputs -----------------------------------------------------------------------------------------------------------------------
def bits(t):
    """t viewed as the integers its sentinel is compared in."""
    return t.view(SENTINEL[t.dtype][0])


def _pattern(dtype, fill):
    return SENTINEL[dtype][1] if fill is None else int(bits(torch.tensor([fill], dtype=dtype))[0])


def guarded(n, dtype, *, head=GUARD, tail=GUARD, fill=None, device='cuda'):
    """(whole buffer, its n elements after `head`): the buffer holds the dtype's SENTINEL bit pattern, or `fill`."""
    buf = torch.empty(head + n + tail, dtype=dtype, device=device)
    bits(buf).fill_(_pattern(dtype, fill))
    return buf, buf[head:head + n]


def untouched(t, fill=None):
    """Per element: t still holds the sentinel (or fill) bit pattern."""
    return bits(t) == _pattern(t.dtype, fill)


def guards_intact(buf, n, *, head=GUARD, fill=None):
    """Nothing before or after the n elements of a guarded buffer was written."""
    return bool(untouched(buf[:head], fill).all()) and bool(untouched(buf[head + n:], fill).all())


def inside(vs, c0, n, lo=0, split=False, device='cuda'):
    """bool [vs]: the elements [c0, c0 + n) of a vs-element row, and [lo + c0, lo + c0 + n) when split."""
    m = torch.zeros(vs, dtype=torch.bool, device=device)
    m[c0:c0 + n] = True
    if split:
        m[lo + c0:lo + c0 + n] = True
    return m


def assert_written(buf, y, vs, mask, tag):
    """y: the guarded output of buf, rows of vs elements; every element of each row under mask is written and nothing else is."""
    if buf.is_cuda:
        torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()), f'{tag}: written outside the output'
    yv = y.view(-1, vs)
    assert not bool(untouched(yv[:, mask]).any()), f'{tag}: an output element was not written'
    assert bool(untouched(yv[:, ~mask]).all()), f'{tag}: written outside its channels'


# ---- pointers --------------------------------------------------------------------------------------------------------------------------------
def at(t, elems=0):
    """The address of element `elems` of t."""
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * elems)


def given(p):
    """A pointer argument is not NULL (capi.ptr(None) is a NULL c_void_p; callers also pass None)."""
    v = p.value if isinstance(p, ctypes.c_void_p) else p
    return v is not None and v != 0


# ---- split fp16 ------------------------------------------------------------------------------------------------------------------------------
def split(v):
    """fp32 -> (hi, lo) fp16: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def split_cat(v):
    """fp32 [..., C] -> fp16 [..., 2C] = [hi | lo]."""
    return torch.cat(split(v), -1).contiguous()


def join(y, c0, n, lo, split=True):
    """fp16 rows -> float64 [..., n] of channels [c0, c0 + n), plus their lo halves at lo + c0 when split."""
    v = y[..., c0:c0 + n].double()
    return v + y[..., lo + c0:lo + c0 + n].double() if split else v


def split_store(v, vs, lo, split, c0=0):
    """fp32 [..., C] -> fp16 [..., vs] rows: hi at channel c0, lo at lo + c0 when split, every other element seeded junk (never read)."""
    g = torch.Generator(device=v.device).manual_seed(int(v.numel()) % 9973)
    out = torch.randn(*v.shape[:-1], vs, generator=g, device=v.device).half()
    C = v.shape[-1]
    hi = v.half()
    out[..., c0:c0 + C] = hi
    if split:
        out[..., lo + c0:lo + c0 + C] = (v - hi.float()).half()
    return out


def hi_w(w):
    """The hi half of a split weight, which is stored x 2^10."""
    return (w * 1024.0).half().double() / 1024.0


def check_split_layout(t):
    """Every stored pair of t = [hi | lo] is hi = fp16(v), lo = fp16(v - hi): |lo| is at most half an fp16 ulp of hi."""
    C = t.shape[-1] // 2
    hi, lo = t[..., :C].float(), t[..., C:].float()
    assert bool((lo.abs() <= hi.abs() * 2.0 ** -11 + 2.0 ** -24).all())


# ---- signatures and recorded calls -----------------------------------------------------------------------------------------------------------
def _capi():
    """The package's C API, imported when a helper first needs it (see the module docstring)."""
    from real3dportrait_b200 import _capi as capi
    return capi


def launch_signature(fn, args):
    """(entry point, non-pointer arguments) with every float argument rounded to fp32, as the C side receives it."""
    return fn, tuple(ctypes.c_float(a).value if isinstance(a, float) else a for a in args)


def call_signature(fn, args, optional=()):
    """A recorded ctypes call -> launch_signature of its non-pointer arguments (capi._SIGNATURES), then whether each pointer at the
    argument positions `optional` is given."""
    capi = _capi()
    types = capi._SIGNATURES[fn][1]
    return launch_signature(fn, [a for a, t in zip(args, types) if t is not capi._P] + [given(args[i]) for i in optional])


class Recorder:
    """Stands in for the library object: passes every call on unchanged and records record(name, args) of each entry point `select`
    accepts.  As a context manager it installs itself as capi._lib, and with ptrs=True wraps capi.ptr to remember the tensor behind each
    pointer (tensor()); both are restored on exit.  With ptrs=True it holds a reference to the latest tensor passed at each address until
    clear(), so the tensors a module passes stay allocated while it records (its allocator cannot hand their addresses out again)."""

    def __init__(self, lib, select, ptrs=False):
        self.lib, self.select, self.ptrs, self.calls, self.tensors = lib, select, ptrs, [], {}

    def record(self, name, args):
        return name, args

    def ptr(self, t, *a, **k):
        if t is not None:                                       # one entry per address, the latest last
            self.tensors.pop(t.data_ptr(), None)
            self.tensors[t.data_ptr()] = t
        return self._ptr(t, *a, **k)

    def tensor(self, p):
        """The latest tensor passed through ptr whose storage holds address p."""
        for t in reversed(self.tensors.values()):
            if t.data_ptr() <= p < t.data_ptr() + t.numel() * t.element_size():
                return t
        raise AssertionError(f'pointer {p:#x} into no tensor the module passed')

    def clear(self):
        self.calls.clear()
        self.tensors.clear()

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not self.select(name):
            return fn

        def call(*args):
            self.calls.append(self.record(name, args))
            return fn(*args)
        return call

    def __enter__(self):
        capi = _capi()
        self._saved = capi._lib, capi.ptr
        self._ptr = capi.ptr
        capi._lib = self
        if self.ptrs:
            capi.ptr = self.ptr
        return self

    def __exit__(self, *exc):
        capi = _capi()
        capi._lib, capi.ptr = self._saved
        return False


# ---- plan assertions ---------------------------------------------------------------------------------------------------------------------------
def assert_plan(got, want, where):
    """The recorded launches equal the plan's; otherwise name what the module launches that the plan lacks, and the reverse."""
    assert got == want, f'{where}: the module launches ' + ('; '.join(f'{x}' for x in got if x not in want) or 'nothing new') + \
        ' not in launch_plan, which has ' + ('; '.join(f'{x}' for x in want if x not in got) or 'nothing more') + \
        f' ({len(got)} launches recorded, {len(want)} planned; where both sets agree, the order differs)'


def assert_rows(missing, stale, label):
    """No launch of `label` lacks a float64 row, and no row it should launch is stale."""
    assert not missing, f'{label} launches without a float64 row:\n' + '\n'.join(missing)
    assert not stale, f'rows {label} no longer launches:\n' + '\n'.join(stale)


# ---- r3dp_mf_conv3d --------------------------------------------------------------------------------------------------------------------------
#: the non-pointer arguments of r3dp_mf_conv3d in C order, as a plan row lists them
CONV3D_ARGS = ('xs', 'xlo', 'cin', 'N', 'D', 'H', 'W', 'kd', 'kh', 'kw', 'up', 'O', 'cop', 'relu', 'ys', 'yc0', 'ylo', 'out_f32', 'split')


def conv3d(a, x, wp, bias, res, y, **override):
    """r3dp_mf_conv3d with a plan row's arguments a (C order), the named ones (N, H, W) replaced.  x, res, y: tensors or pointers (res None:
    no residual)."""
    v = list(a[:len(CONV3D_ARGS)])
    for k, val in override.items():
        v[CONV3D_ARGS.index(k)] = val
    capi = _capi()
    p = lambda t, dt: t if isinstance(t, ctypes.c_void_p) else capi.ptr(t, dt)      # noqa: E731
    capi.check(capi.lib().r3dp_mf_conv3d(p(x, F16), *v[:3], capi.ptr(wp, F16), capi.ptr(bias), p(res, F16), *v[3:14],
                                         p(y, getattr(y, 'dtype', None)), *v[14:], capi.stream()))
