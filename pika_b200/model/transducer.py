"""Generic transducer -- drop-in for trainer/model/transducer.py (reference).

``Net(opt, input_dim, output_dim)`` / ``forward(x, y, x_len, softmax)`` and the sub-module names
``encoder, embed, decoder, fc1, fc_gate, fc2`` are the reference's.  The joint's layers are run by engine.joint_forward /
joint_backward (the MBR trainer too) and, for the graph-replayed beam search, read by the decoder.  Either encoder of the reference: the LSTM (``encoder_type == 'rnn'``, optionally bidirectional,
run over the packed lengths ``x_len``) or the TDNN-Transformer; and either prediction net: the LSTM stack
(``decoder_type == 'rnn'``) or the convolutional transformer (``'transformer'``, trainer/model/rnnt_conv_transformer_lm.py).
Modules are created in the reference's order, so ``torch.manual_seed(s); Net(...)`` draws the reference's initial weights.
"""
import torch.nn as nn

from .rnnt_conv_transformer_lm import Net as decoder_transformer
from .rnnt_tdnn_transformer import Net as encoder_tdnn


def add_simple_joiner(net, hid_dim, output_dim):
    """simple_am_proj / simple_lm_proj: the two linear maps of the simple joiner am[t] + lm[u] (encoder and prediction-net outputs to
    the vocabulary).  Also used to extend a dense checkpoint for pruned training."""
    net.simple_am_proj = nn.Linear(hid_dim, output_dim)
    net.simple_lm_proj = nn.Linear(hid_dim, output_dim)


class Net(nn.Module):
    def __init__(self, opt, input_dim, output_dim):
        super().__init__()
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.hid_dim = opt.rnn_size
        self.local_rank = getattr(opt, "local_rank", 0)
        self.decoder_type = opt.decoder_type
        if opt.encoder_type == "rnn":                  # trainer/model/transducer.py:35-44
            self.encoder = nn.LSTM(input_size=input_dim, hidden_size=self.hid_dim // (2 if opt.brnn else 1), dropout=opt.dropout,
                                   num_layers=opt.enc_layers, bidirectional=bool(opt.brnn), batch_first=True)
            self.pack_seq = True
        else:
            self.encoder = encoder_tdnn(input_dim=input_dim, input_ctx=0, output_dim=self.hid_dim,
                                        tdnn_nhid=1024, tdnn_layers=9)
            self.encoder.chunk_size = getattr(opt, "chunk_size", 0)              # streaming (chunk-limited attention)
            self.encoder.left_chunks = getattr(opt, "left_chunks", -1)
            self.pack_seq = False
        self.embed = nn.Embedding(output_dim + 1, opt.embd_dim, padding_idx=opt.padding_idx)
        if opt.decoder_type == "rnn":
            self.decoder = nn.LSTM(input_size=opt.embd_dim, hidden_size=self.hid_dim, dropout=opt.dropout,
                                   num_layers=opt.dec_layers, bidirectional=False, batch_first=True)
        else:                                          # trainer/model/transducer.py:62-68
            self.decoder = decoder_transformer(embeddings=self.embed, output_dim=self.hid_dim, d_model=512,
                                               num_layers=opt.dec_layers, heads=8, d_ff=2048, dropout=opt.dropout,
                                               max_relative_positions=getattr(opt, "max_relative_positions", 0))
        self.fc1 = nn.Linear(2 * self.hid_dim, self.hid_dim)
        self.fc_gate = nn.Linear(2 * self.hid_dim, self.hid_dim)
        self.fc2 = nn.Linear(self.hid_dim, output_dim)
        if getattr(opt, "prune_range", 0) > 0:
            # the pruned RNN-T loss's simple joiner (engine.transducer_loss_pruned), created after every module of the reference so
            # that a seeded Net still draws the reference's weights for those; forward and decoding never use it
            add_simple_joiner(self, self.hid_dim, output_dim)

    def forward(self, x, y, x_len=None, softmax=True):
        """x [B,T,D] f32, y [B,U] int64 -> [B,T',U+1,V] log-probs (or logits if softmax=False).  With the LSTM encoder, x_len
        packs the batch (T' = max(x_len)); the TDNN-Transformer encoder ignores it."""
        from pika_b200 import engine
        return engine.transducer_forward(self, x, y, softmax, x_len=x_len)

    def clean_hidden(self):
        """interface kept from the reference"""

    def reset_hidden(self, h, reset_idx):
        """interface kept from the reference"""
