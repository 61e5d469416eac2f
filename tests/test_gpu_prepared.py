"""Moving an SR head drops its prepared weights: for the plain head with constant styles, large_sr and the torso head, in `tc` and
`tc_exact`, a `.to(device)` after a forward makes the next forward build new prepared tensors (and drops the torso head's clip constants),
and the image stays bit-identical.  The head is moved to the device it is already on."""
import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda'
N = 2
SR_KW = dict(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True)


def _head(kind, mode):
    if kind == 'plain':
        m, sd = r3.SuperresolutionHybrid8XDC(sr_mode=mode, **SR_KW), syn.make_sr_params(seed=5)
    elif kind == 'large':
        m, sd = r3.SuperresolutionHybrid8XDC(large_sr=True, sr_mode=mode, resblocks_in_large_sr=2, **SR_KW), syn.make_sr_large_params(seed=8, n_res=2)
    else:
        m = r3.SuperresolutionHybrid8XDC_Warp(sr_mode=mode, hp=syn.WARP_HPARAMS, torso_model=syn.StubTorsoModel(), **SR_KW)
        sd = syn.make_sr_warp_params(seed=6)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV).eval()
    m.static_styles = True                                             # the styles below are all ones
    return m


def _args(kind):
    g = torch.Generator().manual_seed(11)
    x = (torch.rand(N, 32, 128, 128, generator=g) * 2 - 1).to(DEV)
    args = (x[:, :3].contiguous(), x, torch.ones(N, 14, 512, device=DEV))
    if kind != 'torso':
        return args
    inp = {k: v.expand(N, *v.shape[1:]).contiguous().to(DEV) for k, v in syn.make_warp_inputs(1, seed=12).items()}
    kp_d = (torch.rand(N, 68, 3, generator=g) * 2 - 1).to(DEV)
    return args + (inp['ref_torso_rgb'], inp['ref_bg_rgb'], torch.rand(N, 1, 128, 128, generator=g).to(DEV), inp['segmap'], inp['kp_s'], kp_d)


def _image(m, args):
    out = m(*args, noise_mode='none')
    return (out[0] if isinstance(out, tuple) else out).clone()


def _tensors(v):
    if isinstance(v, torch.Tensor):
        yield v
    elif isinstance(v, dict):
        for x in v.values():
            yield from _tensors(x)
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _tensors(x)
    else:
        for s in getattr(v, '__slots__', ()):                           # sr_tc.Prepared
            yield from _tensors(getattr(v, s))


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
@pytest.mark.parametrize('kind', ['plain', 'large', 'torso'])
def test_move_rebuilds_prepared_weights(kind, mode):
    m, args, split = _head(kind, mode), _args(kind), mode == 'tc_exact'
    names = {'plain': ['styles'], 'large': ['styles', 'large'], 'torso': ['styles', 'plain']}[kind]
    with torch.no_grad():
        if kind == 'torso':
            m.begin_clip(args[3][:1], args[4][:1], batch=N)
        first = _image(m, args)
        before = {n: m.cached(n, split) for n in names}
        m.to(DEV)
        assert all(m.cached(n, split) is None for n in names)
        if kind == 'torso':
            assert m._clip_cache is None                               # moved mid-clip: uncached until the next begin_clip
        again = _image(m, args)
    for n in names:
        old, new = list(_tensors(before[n])), list(_tensors(m.cached(n, split)))
        assert old and len(new) == len(old), n
        assert not {id(t) for t in old} & {id(t) for t in new}, n
    assert torch.equal(again, first)
