"""FrameEngine(out_mode='concat_debug') rejections that need no GPU: each is raised before the engine touches a device."""
import pytest
import torch

from real3dportrait_b200 import engine


def test_out_mode_rejections():
    bb = torch.nn.Module()
    with pytest.raises(ValueError, match='out_mode'):
        engine.FrameEngine(out_mode='debug')
    with pytest.raises(ValueError, match='secc2plane'):
        engine.FrameEngine(out_mode='concat_debug', out_uint8=True)
    with pytest.raises(ValueError, match='out_uint8'):
        engine.FrameEngine(out_mode='concat_debug', secc2plane=bb)
    for exchange in ('allgather', 'none'):
        with pytest.raises(NotImplementedError, match='p2p'):
            engine.FrameEngine(out_mode='concat_debug', secc2plane=bb, out_uint8=True, world=2, rank=0, exchange=exchange)
    with pytest.raises(NotImplementedError, match='mask_invalid_rays'):
        engine.FrameEngine(out_mode='concat_debug', secc2plane=bb, out_uint8=True, hp={'mask_invalid_rays': True})
