"""Convolutional-transformer prediction net -- drop-in for trainer/model/rnnt_conv_transformer_lm.py (reference).

Same constructor signature, attribute names and state_dict keys (``embeddings, conv.N, transformer.N.{self_attn.*,
feed_forward.*, layer_norm}, layer_norm, linear_out`` and the ``mask`` buffer), created in the reference's order so that a
seeded construction yields its initial weights bit for bit.  ``forward`` runs on the sm_90a kernels
(pika_b200/engine.py:conv_transformer_lm_forward_act): the causal convolution is one GEMM over overlapping activation rows,
the self-attention uses the masked softmax kernel (causal + padding keys; the relative-position band kernels when
``max_relative_positions`` > 0), everything else is the encoder's transformer layer.
"""
import numpy as np
import torch
import torch.nn as nn

from .rnnt_tdnn_transformer import _TransformerLayerParams


class Net(nn.Module):
    """trainer/model/rnnt_conv_transformer_lm.py:12-87"""

    def __init__(self, embeddings, output_dim, d_model, num_layers, heads=8, d_ff=2048, dropout=0.1, max_relative_positions=0,
                 max_size=5000):
        super().__init__()
        self.embeddings = embeddings
        self.output_dim = output_dim
        self.max_relative_positions = max_relative_positions
        self.conv = nn.ModuleList(
            [nn.Conv1d(embeddings.embedding_dim, d_model, kernel_size=5, padding=4)] +
            [nn.Conv1d(d_model, d_model, kernel_size=5, padding=4) for _ in range(num_layers - 1)])
        self.transformer = nn.ModuleList([_TransformerLayerParams(d_model, heads, d_ff, dropout, max_relative_positions)
                                          for _ in range(num_layers)])
        self.layer_norm = nn.LayerNorm(d_model, eps=1e-6)
        self.linear_out = nn.Linear(d_model, output_dim)
        # kept for state_dict compatibility (:56-58, 82-87); the kernels build the causal mask from the row index
        self.register_buffer("mask", torch.from_numpy(np.triu(np.ones((1, max_size, max_size)), k=1).astype("uint8")))

    def forward(self, src, softmax=False):
        """src [B, L] int64 -> [B, L, output_dim] f32 (log-probs when ``softmax``)"""
        from pika_b200 import engine
        out = engine.conv_transformer_lm_forward_act(self, src).float()
        if softmax:
            out = torch.log_softmax(out, dim=-1)       # not used by the transducer (trainer/model/transducer.py:96-97 passes the default)
        return out
