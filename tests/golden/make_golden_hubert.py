"""Writes hubert_small.npz from the reference's own extract_hubert.get_hubert_from_16k_speech, run in float64 on a seeded small HubertModel of
the built architecture (conv_dim 32 x 7, hidden 128, 2 heads, FFN 256, 2 layers, pos conv k128 in 2 groups), with a local
Wav2Vec2FeatureExtractor(do_normalize=True).  Needs the reference tree and transformers; nothing is downloaded.
Usage: python tests/golden/make_golden_hubert.py /path/to/reference"""
import os
import sys
import types

import numpy as np
import torch

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get('R3DP_REFERENCE', '/root/reference')
sys.path.insert(0, REF)
from transformers import HubertConfig, HubertModel, Wav2Vec2FeatureExtractor  # noqa: E402
sys.modules['soundfile'] = types.ModuleType('soundfile')          # only the wav-file path reads it
import data_gen.utils.process_audio.extract_hubert as eh  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hubert_reference import formula_params, wave  # noqa: E402

SMALL = dict(conv_dim=(32,) * 7, hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=2,
             num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=2, feat_extract_norm='layer', do_stable_layer_norm=True,
             conv_bias=True, feat_proj_layer_norm=True)
LARGE = dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
             num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
             conv_bias=True, feat_proj_layer_norm=True)


class Double(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, x):
        return self.m(x.double())


def main():
    m = HubertModel(HubertConfig(**SMALL)).double().eval()
    vals = formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict(vals, strict=True)
    eh.hubert_model = Double(m)
    eh.wav2vec2_processor = Wav2Vec2FeatureExtractor(do_normalize=True, return_attention_mask=False)
    out = {'config.' + k: np.array(v) for k, v in SMALL.items()}
    for L in (400, 4000, 330000):
        out[f'hubert_{L}'] = eh.get_hubert_from_16k_speech(wave(L), device='cpu').numpy().astype(np.float32)
    # the T the reference returns at chunk-boundary lengths (a zero-layer encoder: only the shapes matter)
    eh.hubert_model = Double(HubertModel(HubertConfig(**dict(SMALL, num_hidden_layers=0))).double().eval())
    lens = [320000 + d for d in range(-3, 4)] + [320080, 320399, 320400, 640079]
    out['T_lens'] = np.array(lens)
    out['T_ref'] = np.array([eh.get_hubert_from_16k_speech(np.sin(np.arange(L) * 0.01).astype(np.float32), device='cpu').shape[0] for L in lens])
    big = HubertModel(HubertConfig(**LARGE))
    keys = list(big.state_dict().keys())
    out['large_keys'] = np.array(keys)
    out['large_shapes'] = np.array([','.join(map(str, v.shape)) for v in big.state_dict().values()])
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'hubert_small.npz'), **out)


if __name__ == '__main__':
    main()
