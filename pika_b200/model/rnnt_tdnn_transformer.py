"""TDNN-Transformer encoder -- drop-in for trainer/model/rnnt_tdnn_transformer.py (reference).

Same constructor signature, attribute names and state_dict keys (``fc_in, bn_in, hidden_conv.N,
hidden_bn.N, transformer.N.{self_attn.{linear_keys,linear_values,linear_query,final_linear},
feed_forward.{w_1,w_2,layer_norm}, layer_norm}, bn_final, fc_out``), created in the same order so
that a seeded construction yields the reference's initial weights bit for bit.  The parameters
live in ordinary torch containers; ``forward`` runs on the hand-written sm_90a kernels
(pika_b200/engine.py) -- there is no torch-op compute path.
"""
import math

import torch.nn as nn


class _AttnParams(nn.Module):
    """trainer/model/modules/multi_headed_attn.py:85-108 (parameter layout only).  ``max_relative_positions`` m > 0 adds the
    relative-position table ``relative_positions_embeddings`` = nn.Embedding(2m+1, dim_per_head), created right after
    ``final_linear`` as in the reference (:103-108)."""

    def __init__(self, head_count, model_dim, dropout, max_relative_positions=0):
        super().__init__()
        assert model_dim % head_count == 0
        self.dim_per_head = model_dim // head_count
        self.model_dim = model_dim
        self.head_count = head_count
        self.linear_keys = nn.Linear(model_dim, model_dim)
        self.linear_values = nn.Linear(model_dim, model_dim)
        self.linear_query = nn.Linear(model_dim, model_dim)
        self.dropout_p = dropout
        self.final_linear = nn.Linear(model_dim, model_dim)
        self.max_relative_positions = max_relative_positions
        if max_relative_positions > 0:
            self.relative_positions_embeddings = nn.Embedding(2 * max_relative_positions + 1, self.dim_per_head)


class _FfnParams(nn.Module):
    """trainer/model/modules/position_ffn.py:16-25 (parameter layout only)."""

    def __init__(self, d_model, d_ff, dropout):
        super().__init__()
        self.w_1 = nn.Linear(d_model, d_ff)
        self.w_2 = nn.Linear(d_ff, d_model)
        self.layer_norm = nn.LayerNorm(d_model, eps=1e-6)
        self.dropout_p = dropout


class _TransformerLayerParams(nn.Module):
    """trainer/model/modules/transformer.py:74-83 (parameter layout only)."""

    def __init__(self, d_model, heads, d_ff, dropout, max_relative_positions=0):
        super().__init__()
        self.self_attn = _AttnParams(heads, d_model, dropout, max_relative_positions)
        self.feed_forward = _FfnParams(d_model, d_ff, dropout)
        self.layer_norm = nn.LayerNorm(d_model, eps=1e-6)
        self.dropout_p = dropout


class Net(nn.Module):
    """Encoder: fc_in+ReLU+BN -> 9 x (TDNN(3 taps)+ReLU+BN), a Transformer layer after TDNN 3/6/9,
    last TDNN stride 4 -> BN -> fc_out (trainer/model/rnnt_tdnn_transformer.py:27-89)."""

    TDNN_DIL_STRIDE = [(1, 1)] * 3 + [(3, 1)] * 5 + [(3, 4)]
    HEADS = [16, 16, 8]
    XF_DROPOUT = 0.2        # hard-wired in the reference (:65)
    # streaming (DESIGN.md "Chunked attention"): chunk width in output frames (0 = full context) and how many earlier chunks a frame
    # may attend to (-1 = all).  Plain attributes, not state: state_dict keys do not change, and pickles without them read these.
    chunk_size = 0
    left_chunks = -1

    def __init__(self, input_dim, input_ctx, output_dim, tdnn_nhid, tdnn_layers, bn_dim=0):
        super().__init__()
        assert tdnn_layers == 9, "the reference encoder is only defined for 9 TDNN layers"
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.tdnn_nhid = tdnn_nhid
        self.filter_size = 3
        self.fc_in = nn.Linear(input_dim, tdnn_nhid)
        self.bn_in = nn.BatchNorm1d(tdnn_nhid)
        self.hidden_conv = nn.ModuleList(
            [nn.Conv2d(1, tdnn_nhid, kernel_size=(3, tdnn_nhid), dilation=(d, 1), stride=(s, 1))
             for (d, s) in self.TDNN_DIL_STRIDE])
        self.hidden_bn = nn.ModuleList([nn.BatchNorm1d(tdnn_nhid) for _ in range(tdnn_layers)])
        self.transformer = nn.ModuleList(
            [_TransformerLayerParams(tdnn_nhid, self.HEADS[i], tdnn_nhid * 4, self.XF_DROPOUT) for i in range(3)])
        self.bn_final = nn.BatchNorm1d(tdnn_nhid)
        self.fc_out = nn.Linear(tdnn_nhid, output_dim)

    def attention_geometry(self):
        """[(s_l, o_l)] of the attention layers: frame i of attention layer l reads input frames up to s_l * i + o_l (each TDNN is a
        valid convolution: output i reads inputs s*i + k*d, k < filter_size)"""
        geo, s, o = [], 1, 0
        for l, (dil, stride) in enumerate(self.TDNN_DIL_STRIDE):
            o += s * (self.filter_size - 1) * dil
            s *= stride
            if (l + 1) % 3 == 0:
                geo.append((s, o))
        return geo

    def chunk_masks(self, chunk_size=None, left_chunks=None):
        """per attention layer, the chunk mask (chunk_len, chunk_off, left_chunks) of ``chunk_size`` output frames (default: the
        attributes), or None everywhere for full context.  A frame belongs to the chunk that holds its rightmost input frame, so a chunk
        of C output frames is W = C * (product of the strides) input frames, and layer l's frame i is in chunk (i + o_l // s_l) //
        (W // s_l)."""
        C = self.chunk_size if chunk_size is None else int(chunk_size)
        left = self.left_chunks if left_chunks is None else int(left_chunks)
        if C < 0 or left < -1:
            raise ValueError("chunk_size must be >= 0 and left_chunks >= -1 (got %d, %d)" % (C, left))
        geo = self.attention_geometry()
        if C == 0:
            return [None] * len(geo)
        W = C * math.prod(stride for _, stride in self.TDNN_DIL_STRIDE)
        return [(W // s, o // s, left) for s, o in geo]

    def forward(self, x, frame_offset=0):
        from pika_b200 import engine
        return engine.encoder_forward(self, x)[:, frame_offset:, :]
