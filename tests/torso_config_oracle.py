"""CPU oracle of the torso head's configurations beside the weighted fuse modes of oracle/real3d_oracle.py::superres_warp, restated from that
module's building blocks: weight_fuse=False (modules/real3d/super_resolution/sr_with_ref.py:158-161) and torso_model_version 'v1' (:84-85)."""
import torch

from oracle import real3d_oracle as orc


def superres_warp(rgb, x, ws, ref_torso_rgb, ref_bg_rgb, weights_img, segmap, kp_s, kp_d, p, torso_model, head_threshold=0.9, mode='v2',
                  weight_fuse=True, torso_version='v2'):
    """SuperresolutionHybrid8XDC_Warp.forward, eval mode.  weight_fuse=False: cat[x, x_torso, x_bg] unweighted -> fuse_fg_bg_convs -> block1 without a
    skip image (`mode` ignored).  torso_version 'v1' calls the warper without the head weights image; nothing else in the head changes."""
    if torso_version == 'v1':
        v1 = torso_model
        torso_model = lambda t, s, ks, kd, h, w, **kw: v1(t, s, ks, kd, h, **kw)           # noqa: E731
    if weight_fuse:
        return orc.superres_warp(rgb, x, ws, ref_torso_rgb, ref_bg_rgb, weights_img, segmap, kp_s, kp_d, p, torso_model, head_threshold, mode)
    ws3 = ws[:, -1:, :].expand(rgb.shape[0], 3, -1)
    if x.shape[-1] != 128:
        x, rgb = orc.resize_bilinear(x, 128), orc.resize_bilinear(rgb, 128)
    rgb_256 = orc.resize_bilinear(rgb, 256)
    weights_256 = orc.resize_bilinear(weights_img, 256)
    ref_torso_256, ref_bg_256 = orc.aa_down2(ref_torso_rgb), orc.aa_down2(ref_bg_rgb)
    x, _ = orc.synthesis_block(x, rgb, ws3, p, 'block0.')
    _, ret = torso_model(ref_torso_256, segmap, kp_s, kp_d, rgb_256, weights_256, cal_loss=True, target_torso_mask=None)
    x_torso = orc.conv_plain(ret['deformed_torso_hid'], p, 'torso_encoder.0')
    x_bg = orc.conv_plain(orc.conv_plain(orc.conv_plain(ref_bg_256, p, 'bg_encoder.0', 0.01), p, 'bg_encoder.2', 0.01), p, 'bg_encoder.4')
    x = torch.cat([x, x_torso, x_bg], dim=1)
    x = orc.conv_plain(orc.conv_plain(orc.conv_plain(x, p, 'fuse_fg_bg_convs.0', 0.01), p, 'fuse_fg_bg_convs.2', 0.01), p, 'fuse_fg_bg_convs.4')
    x = orc.synthesis_layer(x, ws3[:, 0], p, 'block1.conv0.', up=2)
    x = orc.synthesis_layer(x, ws3[:, 1], p, 'block1.conv1.', up=1)
    return orc.to_rgb(x, ws3[:, 2], p, 'block1.torgb.'), ret
