#!/usr/bin/env python
"""Generate tests/golden/decode_xf_fst.npz by EXECUTING THE REFERENCE's own TransducerDecoder with the convolutional-transformer
prediction net and on-the-fly FST shallow fusion (lm_scorer = the reference's own SortedMatcher, decoder/sorted_matcher.py, over the
toy back-off LM of make_inputs.py held in make_golden.py's in-memory stand-in for the PyKaldi VectorFst), imported through
tests/golden/ref_shim.py.

Model and encoder outputs are those of decode_xf.npz (make_golden.py:golden_decode_xf); lm_scorer_scale 0.5, nonblk_reward 0.45 as in
decode_fst.npz; beam 4 / n-best 2 and beam 8 / n-best 4 with max_relative_positions 0, and beam 4 / n-best 2 with
max_relative_positions 4 (the model of make_golden_relpos.py:golden_decode_xf_relpos).

Run on the CPU, next to the reference checkout ref_shim.py imports:   python tests/golden/make_golden_xf_fst.py
No test runs this script; the tests read the .npz it writes.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import _FakeFst, build_ref_model_xf, ref_shim, xf_inputs  # noqa: E402  (installs the reference shim)
from make_golden_relpos import build_ref_model_xf_relpos  # noqa: E402

# (case name, beam, n_best, max_relative_positions)
CASES = [("b4n2", 4, 2, 0), ("b8n4", 8, 4, 0), ("rel4_b4n2", 4, 2, 4)]
SEED = 808
V, B, Tp = 40, 4, 24
TLENS = [24, 21, 17, 9]


def golden_decode_xf_fst():
    ref_shim.load_beam_module()
    from decoder.transducer_decoder import TransducerDecoder
    from decoder.sorted_matcher import SortedMatcher
    import decoder.beam_transducer as bt
    from fixture_utils import decode_fixture_reinit_xf
    from make_inputs import toy_backoff_lm
    arcs, finals = toy_backoff_lm(V)
    matcher = SortedMatcher(_FakeFst(arcs, finals), max(len(a) for a in arcs), V + 2, 1, [])
    enc_t = torch.from_numpy(xf_inputs(SEED, B, Tp))

    class FixedEncoder(torch.nn.Module):
        def forward(self, x):
            return enc_t

    tl = torch.tensor(TLENS)
    cases = {}
    saved = torch.cuda.LongTensor
    torch.cuda.LongTensor = torch.LongTensor          # the reference's transformer branch builds torch.cuda.LongTensor (:166)
    try:
        for name, beam, nbest, m_rel in CASES:
            m = build_ref_model_xf(V) if m_rel == 0 else build_ref_model_xf_relpos(V, m_rel)
            m.eval()
            decode_fixture_reinit_xf(m)
            m.encoder = FixedEncoder()
            dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.45)
            dec = TransducerDecoder(m, B, beam, n_best=nbest, blk=0, global_scorer=bt.GlobalScorer(), sm_scale=1.0, cuda=False,
                                    lm_scorer=matcher, lm_scorer_scale=0.5, beam_prune=True, args=dargs)
            with torch.no_grad():
                ret, _ = dec.decode_batch(torch.zeros(B, 1, 240), tl, max_len=[int(t) + 30 for t in tl])
            for b in range(B):
                for n in range(nbest):
                    cases["%s_pred_%d_%d" % (name, b, n)] = np.array([int(t) for t in ret["predictions"][b][n]], np.int64)
                    cases["%s_score_%d_%d" % (name, b, n)] = np.array(float(ret["scores"][b][n]))
            print("decode_xf_fst", name, [[int(t) for t in cases["%s_pred_%d_0" % (name, b)] if t != 0] for b in range(B)],
                  [round(float(cases["%s_score_%d_0" % (name, b)]), 3) for b in range(B)])
    finally:
        torch.cuda.LongTensor = saved
    np.savez_compressed(os.path.join(HERE, "decode_xf_fst.npz"), seed=np.array(SEED), tlens=tl.numpy(), dims=np.array([V, B, Tp]),
                        cases=np.array([c[0] for c in CASES]), beams=np.array([c[1] for c in CASES]),
                        nbests=np.array([c[2] for c in CASES]), rel_m=np.array([c[3] for c in CASES]), **cases)


if __name__ == "__main__":
    golden_decode_xf_fst()
