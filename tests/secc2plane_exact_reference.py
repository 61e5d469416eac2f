"""The launch sequence of SegFormerSECC2PlaneBackbone(precision='tc_exact'), restated from the architecture (MiT-b0 stages, SegFormerHead,
to_plane_cnn) and the split-operand rule rather than from the module's code, and the float64 weight packing the module must produce.

Rule: every GEMM / conv operand is split fp16 (three MMAs); every activation the `tc` plan (secc2plane_reference.launch_plan) passes between
launches as fp16 is passed as fp32 (the GEMM outputs the attention and the DWConv read) or as split rows [hi C | lo C].

exact_flow(H, B) lists each launch as (tag, C entry point, the non-pointer arguments in C order, reads, writes), reads / writes being
(buffer, form, row width) with form 'f32' (rows of width floats) or 'split' (rows of 2 width halves, hi then lo); launch_plan_exact drops the
buffer columns, in secc2plane_reference.launch_plan's format."""
import torch

import secc2plane_reference as ref
from secc2plane_reference import EMB, EMBED, HEADS, SR, cop_of

SPLIT_ENTRY_POINTS = ('r3dp_sp_layernorm_split', 'r3dp_sp_patches_split', 'r3dp_sp_attention_split', 'r3dp_sp_dwconv_gelu_split',
                      'r3dp_sp_head_fuse_split', 'r3dp_sp_leaky_split', 'r3dp_sp_upsample2_flip_split')


def exact_flow(H, B, cin=9):
    rows = []

    def add(tag, fn, args, reads, writes):
        rows.append((tag, fn, tuple(args), tuple(reads), tuple(writes)))

    def gemm(tag, src, R, K, O, dst):
        """split operands (xs = 2K, xlo = K), fp32 out"""
        add(tag, 'r3dp_mf_conv3d', (2 * K, K, K, 1, 1, 1, R, 1, 1, 1, 0, O, cop_of(O), 0, O, 0, 0, 1, 1), [(src, 'split', K)], [(dst, 'f32', O)])

    h = (H - 1) // 4 + 1
    add('embed', 'r3dp_sp_embed', (B, cin, H, H), [('x', 'f32', cin)], [('t0', 'f32', EMBED[0])])
    levels = []
    prev = None
    for s in range(4):
        C, st = EMBED[s], f's{s + 1}'
        if s > 0:
            add(st + '.pe_patches', 'r3dp_sp_patches_split', (B, h, h, EMBED[s - 1], 3, 2, 1), [(prev, 'split', EMBED[s - 1])],
                [(st + '.pt', 'split', 9 * EMBED[s - 1])])
            h = (h + 2 - 3) // 2 + 1
            gemm(st + '.pe', st + '.pt', B * h * h, 9 * EMBED[s - 1], C, 't0')
        R = B * h * h
        add(st + '.pe_norm', 'r3dp_sp_layernorm', (R, C, 1e-5, C), [('t0', 'f32', C)], [(st + '.x', 'f32', C)])
        add(st + '.norm1', 'r3dp_hb_layernorm', (R, C, 1e-6, 0, 0, 2 * C, C), [(st + '.x', 'f32', C)], [(st + '.a', 'split', C)])
        for bi in range(2):
            gemm(st + '.q', st + '.a', R, C, C, 'q')
            if SR[s] > 1:
                k = SR[s]
                hk = h // k
                add(st + '.sr_patches', 'r3dp_sp_patches_split', (B, h, h, C, k, k, 0), [(st + '.a', 'split', C)], [(st + '.srpt', 'split', k * k * C)])
                gemm(st + '.sr', st + '.srpt', B * hk * hk, k * k * C, C, 'r')
                add(st + '.sr_norm', 'r3dp_hb_layernorm', (B * hk * hk, C, 1e-5, 0, 0, 2 * C, C), [('r', 'f32', C)], [(st + '.a2', 'split', C)])
                gemm(st + '.kv', st + '.a2', B * hk * hk, C, 2 * C, 'kv')
                tk = hk * hk
            else:
                gemm(st + '.kv', st + '.a', R, C, 2 * C, 'kv')
                tk = h * h
            add(st + '.attention', 'r3dp_sp_attention_split', (C, 2 * C, B, h * h, tk, HEADS[s], 32 ** -0.5, 2 * C, C),
                [('q', 'f32', C), ('kv', 'f32', 2 * C)], [('o', 'split', C)])
            gemm(st + '.proj', 'o', R, C, C, 't')
            add(st + '.norm2', 'r3dp_sp_layernorm_split', (R, C, 1e-6, 2 * C, C), [(st + '.x', 'f32', C), ('t', 'f32', C)],
                [(st + '.x', 'f32', C), (st + '.a', 'split', C)])
            gemm(st + '.fc1', st + '.a', R, C, 4 * C, 'f1')
            add(st + '.dwconv', 'r3dp_sp_dwconv_gelu_split', (B, h, h, 4 * C), [('f1', 'f32', 4 * C)], [('f2', 'split', 4 * C)])
            gemm(st + '.fc2', 'f2', R, 4 * C, C, 't')
            if bi == 0:
                add(st + '.norm1', 'r3dp_sp_layernorm_split', (R, C, 1e-6, 2 * C, C), [(st + '.x', 'f32', C), ('t', 'f32', C)],
                    [(st + '.x', 'f32', C), (st + '.a', 'split', C)])
            else:
                prev = f'c{s + 1}'
                add(st + '.norm', 'r3dp_sp_layernorm_split', (R, C, 1e-6, 2 * C, C), [(st + '.x', 'f32', C), ('t', 'f32', C)], [(prev, 'split', C)])
        levels.append(h)
    for i, hh in enumerate(levels):
        gemm(f'G{i + 1}', f'c{i + 1}', B * hh * hh, EMBED[i], EMB, f'g{i + 1}')
    h1 = levels[0]
    add('head_fuse', 'r3dp_sp_head_fuse_split', (levels[0], levels[1], levels[2], levels[3], B), [(f'g{i + 1}', 'f32', EMB) for i in range(4)],
        [('y0', 'split', EMB)])
    for j, i in enumerate((0, 2, 4)):
        src, dst = f'y{j}', f'y{j + 1}'
        if h1 % 128 == 0:
            add(f'to_plane_cnn.{i}', 'r3dp_sr_tcx_conv', (B, 1, EMB, EMB, h1, h1, 3, 2), [(src, 'split', EMB)], [(dst, 'split', EMB)])
        else:
            add(f'to_plane_cnn.{i}', 'r3dp_mf_conv3d', (2 * EMB, EMB, EMB, B, 1, h1, h1, 1, 3, 3, 0, EMB, EMB, 0, 2 * EMB, 0, EMB, 0, 1),
                [(src, 'split', EMB)], [(dst, 'split', EMB)])
            add(f'to_plane_cnn.{i + 1}', 'r3dp_sp_leaky_split', (B * h1 * h1, EMB, 0.01), [(dst, 'split', EMB)], [(dst, 'split', EMB)])
    add('upsample', 'r3dp_sp_upsample2_flip_split', (B, h1, h1, EMB), [('y3', 'split', EMB)], [('ur', 'split', EMB), ('urc', 'split', EMB)])
    for O, c0, src in ((64, 0, 'ur'), (32, 64, 'urc')):
        add(f'to_plane_cnn.7[{c0}:{c0 + O}]', 'r3dp_mf_conv3d', (2 * EMB, EMB, EMB, B, 1, 2 * h1, 2 * h1, 1, 3, 3, 0, O, cop_of(O), 0, 96, c0, 0, 1, 1),
            [(src, 'split', EMB)], [('planes', 'f32', 96)])
    return rows


def launch_plan_exact(H, B, cin=9):
    """exact_flow without the buffer columns: (tag, C entry point, non-pointer arguments), as secc2plane_reference.launch_plan."""
    return [r[:3] for r in exact_flow(H, B, cin)]


# ---- the float64 packing ---------------------------------------------------------------------------------------------------------------
def split_rows(w):
    """float64 [..., K] -> fp16 [..., 2K] = [hi | lo] of w * 2^10."""
    s = w * 1024.0
    hi = s.half()
    return torch.cat([hi, (s - hi.double()).half()], -1)


def padded(w, cop):
    """[O, ...] -> [cop, ...] with zero rows after O."""
    out = torch.zeros(cop, *w.shape[1:], dtype=w.dtype)
    out[:w.shape[0]] = w
    return out


def exact_packs(sd):
    """{name: fp16 packed rows} for every r3dp_mf_conv3d weight of the module in tc_exact, from a float64 state_dict with the reference's
    keys: Linear weights [O, K], conv weights as rows (ky, kx, c), the head maps G_i = diag(s) W_fuse,i W_lin,i with the eval BatchNorm's
    s = gamma / sqrt(var + eps), the 3x3 convs as [9, cop, 2I] (tap ky*3 + kx), the last conv's mirrored taps."""
    out = {}

    def gemm(name, w):
        out[name] = split_rows(padded(w, cop_of(w.shape[0])))

    def taps(name, w):
        out[name] = split_rows(padded(w, cop_of(w.shape[0])).permute(2, 3, 0, 1).reshape(9, cop_of(w.shape[0]), w.shape[1]))

    for s in range(4):
        mv = f'mix_vit.block{s + 1}'
        if s > 0:
            w = sd[f'mix_vit.patch_embed{s + 1}.proj.weight']
            gemm(f's{s + 1}.pe', w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))
        for bi in range(2):
            p = f'{mv}.{bi}'
            for n in ('attn.q', 'attn.kv', 'attn.proj', 'mlp.fc1', 'mlp.fc2'):
                gemm(f's{s + 1}.{bi}.{n}', sd[f'{p}.{n}.weight'])
            if SR[s] > 1:
                w = sd[f'{p}.attn.sr.weight']
                gemm(f's{s + 1}.{bi}.attn.sr', w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))
    bn = 'fuse_head.linear_fuse.bn'
    sc = sd[bn + '.weight'] / torch.sqrt(sd[bn + '.running_var'] + 1e-5)
    wf = sd['fuse_head.linear_fuse.conv.weight'][:, :, 0, 0]
    for i in range(4):
        blk = sc[:, None] * wf[:, (3 - i) * EMB:(4 - i) * EMB]
        gemm(f'G{i + 1}', blk @ sd[f'fuse_head.linear_c{i + 1}.proj.weight'])
    for i in (0, 2, 4):
        taps(f'to_plane_cnn.{i}', sd[f'to_plane_cnn.{i}.weight'])
    w7 = sd['to_plane_cnn.7.weight']
    taps('last_r', w7[:64].flip(2))
    taps('last_rc', w7[64:].flip(2, 3))
    return out


__all__ = ['exact_flow', 'launch_plan_exact', 'exact_packs', 'split_rows', 'SPLIT_ENTRY_POINTS', 'ref']
