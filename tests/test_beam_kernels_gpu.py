"""The device beam-search kernels (pika_b200/csrc/beam.cu) called directly through the C ABI.

pk_beam_advance / pk_beam_advance_lm run on an arbitrary state written into device buffers and are compared, every buffer bit for
bit, with the one-step layout oracle (tests/beam_step_oracle.py, pinned to oracle.decode.Beam.advance by test_beam_step_cpu.py).
The oracle is given pk_log_softmax's output for the very logits the kernel reads, so equal scores also check that the kernel's
on-the-fly log-prob is pk_log_softmax's.  Every buffer has a guard region past its end that must keep its sentinel.
Cases: every beam width (1, 2, 4, 8, 16) at one, two and three candidate batches per row (V up to 12289), the scalar load paths,
batch 1 to 70, three softmax scales, step 0 and later steps, chained steps, the kill paths (finished rows, duplicates of 1 to 65
tokens, near-duplicates), the finish rule and its limits, the FST search with disambiguation arcs, a deep back-off chain and
state-set overflow, and the argument checks.  The small step kernels are checked against torch; the transformer prediction net's
single-query attention and conv taps against float64 attention and exact gathers over a scattered slot table; whole decodes at the
widths and vocabularies the golden fixtures do not reach against oracle.decode.decode_batch."""
import ctypes
import types

import numpy as np
import pytest
import torch

import beam_step_oracle as bso

pytestmark = pytest.mark.gpu

GUARD = 37
SENT_I, SENT_F = -12345, 7.25


def _st():
    return torch.cuda.current_stream().cuda_stream


class Dev:
    """the oracle state in device buffers, each followed by GUARD sentinel elements"""

    def __init__(self, st):
        self.shapes, self.buf = {}, {}
        for k, v in st.items():
            dt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}[v.dtype]
            t = torch.full((v.size + GUARD,), SENT_I if dt == torch.int32 else SENT_F, dtype=dt)
            t[:v.size] = torch.from_numpy(np.ascontiguousarray(v).ravel())
            self.buf[k], self.shapes[k] = t.cuda(), v.shape

    def p(self, k):
        return self.buf[k].data_ptr()

    def read(self):
        out = {}
        for k, t in self.buf.items():
            h = t.cpu().numpy()
            n = int(np.prod(self.shapes[k]))
            g = h[n:]
            assert (g == (SENT_I if t.dtype == torch.int32 else SENT_F)).all(), ("guard region overwritten", k)
            out[k] = h[:n].reshape(self.shapes[k])
        return out


def _same(got, want, what=""):
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), (what, k, got[k].ravel()[:64], want[k].ravel()[:64])


def _logits(rows, V, ldv, offset, rng, scale=3.0, blank_bias=0.0):
    """[rows, V] logits inside a [offset + rows * ldv] buffer -> (buffer, address of row 0, the [rows, V] values)"""
    x = (scale * rng.standard_normal((rows, V))).astype(np.float32)
    x[:, 0] += blank_bias
    buf = torch.full((offset + rows * ldv + GUARD,), -3.0e38, dtype=torch.float32)
    buf[offset:offset + rows * ldv].view(rows, ldv)[:, :V] = torch.from_numpy(x)
    buf = buf.cuda()
    return buf, buf.data_ptr() + 4 * offset, x


def _word_probs(addr, rows, V, ldv, sm_scale):
    """pk_row_lse (what the kernel reads) and pk_log_softmax (what the oracle reads) of the same logits"""
    from pika_b200._lib import PK_F32, check, lib
    lse = torch.empty(rows, device="cuda")
    wp = torch.empty(rows, V, device="cuda")
    check(lib.pk_row_lse(addr, PK_F32, ldv, lse.data_ptr(), rows, V, sm_scale, _st()), "pk_row_lse")
    check(lib.pk_log_softmax(addr, PK_F32, ldv, wp.data_ptr(), rows, V, sm_scale, _st()), "pk_log_softmax")
    return lse, wp.cpu().numpy()


class Fst:
    """fusion_lm on the device (pika SortedMatcher) and in the oracle (oracle.decode.SortedMatcher)"""

    def __init__(self, V, scale=1.0, reward=0.0):
        from oracle.decode import SortedMatcher as OM
        from pika_b200.decoder.sorted_matcher import SortedMatcher
        arcs, finals, bo, dis = bso.fusion_lm(V)
        self.dev = SortedMatcher((arcs, finals), max(len(a) for a in arcs), V + 3, bo, dis)
        self.struct, self.keep = self.dev.device_tables(torch.device("cuda"))
        self.oracle = bso.Lm(OM(arcs, finals, bo, dis), scale, reward)


def _advance(dev, addr, lse, ldv, V, sm_scale, t_idx, nf, ml, step_ctx, n_best, prune, fst=None, ms=None):
    from pika_b200._lib import check, lib
    B, K = dev.shapes["scores"]
    L, cap = dev.shapes["hyp_tok"][3], dev.shapes["fin_score"][1]
    c = (addr, ldv, lse.data_ptr(), sm_scale, t_idx.data_ptr(), nf.data_ptr(), ml.data_ptr(), dev.p("scores"), dev.p("next_ys"),
         dev.p("prev_ks"), dev.p("hyp_tok"), dev.p("hyp_len"), dev.p("fin_score"), dev.p("fin_step"), dev.p("fin_k"), dev.p("fin_count"),
         dev.p("eos_top"), dev.p("done"), dev.p("not_done_total"), B, K, V, L, cap, step_ctx.data_ptr(), 0, n_best, prune)
    if fst is None:
        check(lib.pk_beam_advance(*c, _st()), "pk_beam_advance")
    else:
        check(lib.pk_beam_advance_lm(*c, fst.struct, fst.oracle.scale, fst.oracle.reward, dev.p("set_state"), dev.p("set_cost"),
                                     dev.p("set_n"), dev.p("lm_scores"), ms, dev.p("err"), _st()), "pk_beam_advance_lm")


def _i32(a):
    return torch.as_tensor(np.asarray(a, np.int32)).cuda()


def random_state(B, K, V, step, rng, L=None, cap=None, ms=None, fin_frac=0.2):
    """a state at step ``step`` that a decode could have reached: scores, tokens (some finished), partial hypotheses"""
    S = step + 2
    L = L or S + 2
    cap = cap or S * K
    st = bso.init_state(B, K, S, L, cap, 0, ms)
    if step == 0:
        return st
    po = step & 1
    st["scores"] = -np.sort(rng.uniform(0, 20, (B, K)), 1).astype(np.float32)
    tok = rng.integers(0, V, (B, K))
    tok[rng.uniform(size=(B, K)) < fin_frac] = -1
    st["next_ys"][step] = tok
    st["next_ys"][1:step] = rng.integers(0, V, (step - 1, B, K))
    st["prev_ks"][:step] = rng.integers(0, K, (step, B, K))
    st["hyp_len"][po] = rng.integers(0, min(L, step) + 1, (B, K))
    st["hyp_tok"][po] = rng.integers(1, max(V, 2), (B, K, L))
    st["hyp_tok"][po ^ 1] = rng.integers(1, max(V, 2), (B, K, L))          # stale contents of the other parity
    st["fin_count"] = rng.integers(0, 3, B).astype(np.int32)
    for b in range(B):
        n = int(st["fin_count"][b])
        st["fin_score"][b, :n] = rng.uniform(-30, -1, n)
        st["fin_step"][b, :n] = rng.integers(1, step + 1, n)
        st["fin_k"][b, :n] = rng.integers(0, K, n)
    if ms is not None:
        n = rng.integers(1, ms + 1, (B, K))
        st["set_n"][po] = n
        for b in range(B):
            for k in range(K):
                st["set_state"][po, b, k, :n[b, k]] = rng.permutation(6)[:n[b, k]] if n[b, k] <= 6 else rng.integers(0, 6, n[b, k])
                st["set_cost"][po, b, k, :n[b, k]] = rng.uniform(0, 5, n[b, k])
                st["lm_scores"][b, k] = np.float32(-st["set_cost"][po, b, k, :n[b, k]].min())
    return st


def check_step(st, step, V, rng, ldv=None, offset=0, sm_scale=0.5, t_idx=None, nf=None, ml=None, n_best=2, prune=1, fst=None,
               ms=None, logit_scale=3.0, blank_bias=0.0):
    """one advance on the device against the oracle; -> (device state, oracle state)"""
    B, K = st["scores"].shape
    rows = B * K
    ldv = ldv or V
    nf = nf if nf is not None else rng.integers(1, 40, B)
    ml = ml if ml is not None else np.full(B, 10000)
    t_idx = t_idx if t_idx is not None else np.minimum(rng.integers(0, 40, rows), np.repeat(nf, K) - 1)
    buf, addr, _ = _logits(rows, V, ldv, offset, rng, logit_scale, blank_bias)
    lse, wp = _word_probs(addr, rows, V, ldv, sm_scale)
    dev = Dev(st)
    _advance(dev, addr, lse, ldv, V, sm_scale, _i32(t_idx), _i32(nf), _i32(ml), _i32([step, 1]), n_best, prune, fst, ms)
    want, _ = bso.advance(st, wp, t_idx, nf, ml, step, 0, n_best, prune, fst.oracle if fst else None)
    got = dev.read()
    _same(got, want, (K, V, step))
    return got, want


# ------------------------------------------------------------------------------------------------ widths x vocabulary batches
@pytest.mark.parametrize("V", [None, 40, 6143, 6144, 6145, 12289])
@pytest.mark.parametrize("K", [1, 2, 4, 8, 16])
def test_advance_every_width_and_vocab_batch(K, V):
    """V = K (the smallest allowed), 40; 6143 / 6144 / 6145 around one batch of 12 x 512 candidates per row; 12289 (three batches,
    V % 4 != 0).  The pitch is V rounded up to 4 (16-byte loads where V % 4 == 0), at step 0 and at a later step."""
    V = V or K
    rng = np.random.default_rng(1000 * K + V)
    ldv = (V + 3) // 4 * 4
    for step in (0, 5):
        check_step(random_state(3, K, V, step, rng), step, V, rng, ldv=ldv)


@pytest.mark.parametrize("K", [4, 16])
@pytest.mark.parametrize("V,ldv,offset", [(6145, 6145, 0), (1001, 1001, 0), (300, 4100, 0), (6145, 6148, 1), (12288, 12288, 1)],
                         ids=["odd-ldv-scalar", "odd-small-scalar", "wide-ldv-vector", "offset-scalar", "offset-V%4=0-scalar"])
def test_advance_load_paths(K, V, ldv, offset):
    """ldv % 4 != 0 or a base address off 16 bytes: every load is scalar.  The wide-pitch case (ldv = 4100 for V = 300, aligned) runs
    the 16-byte loads with rows far apart."""
    rng = np.random.default_rng(K + V + ldv + offset)
    check_step(random_state(2, K, V, 3, rng), 3, V, rng, ldv=ldv, offset=offset)


@pytest.mark.parametrize("sm_scale", [1.0, 0.5, 0.3])
@pytest.mark.parametrize("B", [1, 3, 70])
def test_advance_batch_and_softmax_scale(B, sm_scale):
    rng = np.random.default_rng(B * 10 + int(sm_scale * 10))
    for step in (0, 1, 4):
        check_step(random_state(B, 8, 300, step, rng), step, 300, rng, sm_scale=sm_scale)


# ------------------------------------------------------------------------------------------------ kill paths
def test_finished_rows_and_an_utterance_with_every_row_finished():
    """finished rows give V candidates at -1e20; an utterance whose rows all finished takes the tie rule at -1e20 (row 0, tokens
    0..K-1) while the others go on"""
    K, V = 8, 50
    rng = np.random.default_rng(3)
    st = random_state(3, K, V, 4, rng, fin_frac=0.5)
    st["next_ys"][4, 1] = -1
    got, _ = check_step(st, 4, V, rng)
    assert got["prev_ks"][4, 1].tolist() == [0] * K and got["next_ys"][5, 1].tolist() == list(range(K))
    assert (got["scores"][1] == np.float32(-1e20)).all()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 65])
@pytest.mark.parametrize("prune", [1, 0])
def test_duplicate_hypotheses(n, prune):
    """rows 0 and 3 hold the same n tokens (not adjacent): row 3 is killed when pruning; row 1 differs from row 0 in its last token,
    row 2 in its 33rd (n > 32) or first, so neither is a duplicate.  Blank is every row's best label by far, so the new beam holds the blank
    of every row that was not killed."""
    K, V, step = 4, 40, 70
    rng = np.random.default_rng(n + 100 * prune)
    st = random_state(1, K, V, step, rng, L=80, fin_frac=0.0)
    po = step & 1
    h = rng.integers(1, V, n)
    rows = [h.copy() for _ in range(K)]
    rows[1][-1] = h[-1] % (V - 1) + 1
    if n > 32:
        rows[2][32] = (h[32] + 1) % (V - 1) + 1           # not row 1's token either
    else:
        rows[2][0] = (h[0] + 1) % (V - 1) + 1
    for k in range(K):
        st["hyp_tok"][po, 0, k, :n] = rows[k]
    st["hyp_len"][po, 0] = n
    st["next_ys"][step, 0] = rng.integers(1, V, K)
    st["scores"][0] = [-2.0, -1.5, -1.0, -0.5]
    got, _ = check_step(st, step, V, rng, prune=prune, logit_scale=0.1, blank_bias=12.0)     # every live row's blank is in the new beam
    pk = got["prev_ks"][step, 0].tolist()
    assert (3 in pk) == (not prune)
    assert 0 in pk and 1 in pk and 2 in pk


# ------------------------------------------------------------------------------------------------ finish rule and limits
def test_finish_rule_order_eos_top_and_done():
    """Blank is the best label of every row and the rows' scores are close, so the new beam is the rows' blanks in score order.
    u0: rows 1 and 2 are on their last frame (finish, eos_top stays 0); u1: back-pointers reversed, row 0's parent on its last frame
    (eos_top, done); u2: max_len reached, every row finishes; u3: already done, finishes again (not_done_total not decremented)."""
    K, V, step = 4, 40, 6
    rng = np.random.default_rng(9)
    st = random_state(4, K, V, step, rng, fin_frac=0.0)
    st["next_ys"][step] = rng.integers(1, V, (4, K))
    st["hyp_len"][step & 1] = 0
    st["fin_count"][:] = 0
    st["scores"][:] = [[0.0, -0.1, -0.2, -0.3], [-0.3, -0.2, -0.1, 0.0], [0.0, -0.1, -0.2, -0.3], [0.0, -0.1, -0.2, -0.3]]
    st["eos_top"][3], st["done"][3], st["fin_count"][3] = 1, 1, 2
    st["not_done_total"][0] = 3
    nf = np.array([10, 10, 10, 10])
    t_idx = np.full(4 * K, 3)
    t_idx[[1, 2]] = 9                                     # u0 rows 1, 2
    t_idx[K + 3] = 9                                      # u1 row 3 = parent of its new row 0
    t_idx[3 * K] = 9
    ml = np.array([10000, 10000, step + 1, 10000])
    got, _ = check_step(st, step, V, rng, t_idx=t_idx, nf=nf, ml=ml, n_best=1, logit_scale=0.01, blank_bias=12.0)
    assert got["prev_ks"][step].tolist() == [[0, 1, 2, 3], [3, 2, 1, 0], [0, 1, 2, 3], [0, 1, 2, 3]]
    assert got["next_ys"][step + 1].tolist() == [[0, -1, -1, 0], [-1, 0, 0, 0], [-1] * 4, [-1, 0, 0, 0]]
    assert got["fin_count"].tolist() == [2, 1, 4, 3] and got["fin_k"][0, :2].tolist() == [1, 2] and got["fin_k"][2, :4].tolist() == [0, 1, 2, 3]
    assert (got["fin_step"][:3, 0] == step + 1).all()
    assert got["eos_top"].tolist() == [0, 1, 1, 1] and got["done"].tolist() == [0, 1, 1, 1]
    assert got["not_done_total"][0] == 1


def test_small_cap_and_L_saturate():
    """cap = 3 and L = 4: the finished lists and the partial hypotheses stop growing; guard regions keep their sentinels"""
    K, V, step = 8, 40, 9
    rng = np.random.default_rng(11)
    st = random_state(2, K, V, step, rng, L=4, cap=3, fin_frac=0.0)
    st["hyp_len"][step & 1] = 4
    st["fin_count"][:] = [2, 3]
    got, _ = check_step(st, step, V, rng, nf=np.array([5, 5]), t_idx=np.full(2 * K, 4), logit_scale=0.01, blank_bias=3.0)
    assert got["fin_count"].tolist() == [3, 3]
    assert (got["hyp_len"][(step & 1) ^ 1] == 4).all()


def test_dead_step_is_a_noop():
    """step_ctx[1] = 0: every beam kernel returns at once; all buffers byte-identical"""
    from pika_b200._lib import PK_F32, check, lib
    K, V, B, H, E = 4, 40, 2, 64, 16
    rng = np.random.default_rng(12)
    fst = Fst(V)
    st = random_state(B, K, V, 3, rng, ms=4)
    dev = Dev(st)
    rows = B * K
    buf, addr, _ = _logits(rows, V, V, 0, rng)
    lse, _ = _word_probs(addr, rows, V, V, 1.0)
    ctx = _i32([3, 0])
    t_idx, nf, ml = _i32(rng.integers(0, 5, rows)), _i32([5, 5]), _i32([100, 100])
    extra = dict(t=t_idx.clone(), enc_hid=torch.randn(rows, H, device="cuda"), x=torch.randn(rows, H, device="cuda"),
                 h=torch.randn(2, rows, H, device="cuda"), c=torch.randn(2, rows, H, device="cuda"), h2=torch.randn(2, rows, H, device="cuda"),
                 c2=torch.randn(2, rows, H, device="cuda"), t2=_i32(rng.integers(0, 5, rows)), ctx=ctx.clone())
    before = {k: v.clone() for k, v in extra.items()}
    enc, emb, gates = torch.randn(B, 6, H, device="cuda"), torch.randn(V, E, device="cuda"), torch.randn(rows, 4 * H, device="cuda")
    check(lib.pk_beam_prepare(dev.p("next_ys"), ctx.data_ptr(), extra["t"].data_ptr(), enc.data_ptr(), PK_F32, 6, H, extra["enc_hid"].data_ptr(),
                              emb.data_ptr(), E, extra["x"].data_ptr(), H, K, 0, rows, _st()), "prepare")
    check(lib.pk_beam_lstm_cell(gates.data_ptr(), dev.p("next_ys"), ctx.data_ptr(), 0, extra["h"].data_ptr(), PK_F32, extra["c"].data_ptr(),
                                rows, H, _st()), "lstm_cell")
    _advance(dev, addr, lse, V, V, 1.0, t_idx, nf, ml, ctx, 1, 1)
    _advance(dev, addr, lse, V, V, 1.0, t_idx, nf, ml, ctx, 1, 1, fst, 4)
    check(lib.pk_beam_reorder(dev.p("prev_ks"), ctx.data_ptr(), extra["h"].data_ptr(), extra["c"].data_ptr(), extra["t"].data_ptr(),
                              extra["h2"].data_ptr(), extra["c2"].data_ptr(), extra["t2"].data_ptr(), PK_F32, K, H, 2, rows, _st()), "reorder")
    check(lib.pk_beam_step_end(extra["ctx"].data_ptr(), dev.p("not_done_total"), 100, _st()), "step_end")
    _same(dev.read(), st)
    for k, v in before.items():
        assert torch.equal(extra[k], v), k


# ------------------------------------------------------------------------------------------------ chained steps
def _reorder_t(t_idx, prev_ks, K):
    B = len(t_idx) // K
    return t_idx.reshape(B, K)[np.arange(B)[:, None], prev_ks].reshape(-1)


@pytest.mark.parametrize("K,prune", [(1, 1), (2, 1), (16, 1), (8, 0)])
def test_chained_steps(K, prune):
    """prepare -> row_lse -> advance -> reorder -> step_end, as TransducerDecoder._beam_step chains them, with fresh logits every step,
    until every utterance is done; t_idx, the state and the step counter are checked after every step"""
    from pika_b200._lib import PK_F32, check, lib
    B, V, H, E = 3, 50, 32, 8
    rng = np.random.default_rng(K * 7 + prune)
    S = 40
    nf, ml = np.array([4, 7, 9]), np.array([10000, 12, 10000])
    st = bso.init_state(B, K, S, S + 1, S * K, 0)
    dev = Dev(st)
    rows = B * K
    ctx = _i32([0, 1])
    t_dev = [_i32(np.full(rows, -1)), _i32(np.full(rows, -1))]
    h = [torch.zeros(1, rows, H, device="cuda") for _ in range(2)]
    c = [torch.zeros(1, rows, H, device="cuda") for _ in range(2)]
    enc, emb = torch.randn(B, 9, H, device="cuda"), torch.randn(V, E, device="cuda")
    enc_hid, x = torch.empty(rows, H, device="cuda"), torch.empty(rows, 8, device="cuda")
    nf_d, ml_d = _i32(nf), _i32(ml)
    t_idx = np.full(rows, -1)
    step = 0
    while True:
        cur, nxt = step & 1, (step & 1) ^ 1
        check(lib.pk_beam_prepare(dev.p("next_ys"), ctx.data_ptr(), t_dev[cur].data_ptr(), enc.data_ptr(), PK_F32, 9, H, enc_hid.data_ptr(),
                                  emb.data_ptr(), E, x.data_ptr(), 8, K, 0, rows, _st()), "prepare")
        buf, addr, _ = _logits(rows, V, V, 0, rng, 2.0, 3.0)
        lse, wp = _word_probs(addr, rows, V, V, 0.8)
        _advance(dev, addr, lse, V, V, 0.8, t_dev[cur], nf_d, ml_d, ctx, 2, prune)
        check(lib.pk_beam_reorder(dev.p("prev_ks"), ctx.data_ptr(), h[cur].data_ptr(), c[cur].data_ptr(), t_dev[cur].data_ptr(),
                                  h[nxt].data_ptr(), c[nxt].data_ptr(), t_dev[nxt].data_ptr(), PK_F32, K, H, 1, rows, _st()), "reorder")
        check(lib.pk_beam_step_end(ctx.data_ptr(), dev.p("not_done_total"), S - 1, _st()), "step_end")
        t_idx = t_idx + (st["next_ys"][step].reshape(-1) == 0)
        assert t_dev[cur].cpu().numpy().tolist() == t_idx.tolist()
        st, _ = bso.advance(st, wp, t_idx, nf, ml, step, 0, 2, prune)
        t_idx = _reorder_t(t_idx, st["prev_ks"][step], K)
        _same(dev.read(), st, step)
        assert t_dev[nxt].cpu().numpy().tolist() == t_idx.tolist()
        step += 1
        live = st["not_done_total"][0] > 0 and step < S - 1
        assert ctx.cpu().tolist() == [step, int(live)]
        if not live:
            break
    assert step > 5 and (st["done"].all() or step == S - 1) and st["fin_count"].sum() > 0


# ------------------------------------------------------------------------------------------------ FST fusion
@pytest.mark.parametrize("ms", [1, 2, 16])
@pytest.mark.parametrize("scale,reward", [(1.0, 0.0), (0.6, 0.3)])
def test_fst_fusion_chained(ms, scale, reward):
    """the fusion LM (disambiguation arcs, back-off depth 3, repeated labels, a label with no arc, a state with no final) over
    12 chained steps; max_states 1 and 2 overflow (err_flag), 16 does not"""
    K, B, V = 8, 3, 20
    rng = np.random.default_rng(ms * 10 + int(scale * 10))
    fst = Fst(V, scale, reward)
    S = 14
    st = bso.init_state(B, K, S, S + 1, S * K, 0, ms)
    dev = Dev(st)
    nf, ml = np.array([6, 9, 30]), np.array([10000, 10, 10000])
    t_idx = np.full(B * K, -1)
    for step in range(12):
        t_idx = t_idx + (st["next_ys"][step].reshape(-1) == 0)
        buf, addr, _ = _logits(B * K, V, V, 0, rng, 2.0, 0.5)
        lse, wp = _word_probs(addr, B * K, V, V, 1.0)
        _advance(dev, addr, lse, V, V, 1.0, _i32(t_idx), _i32(nf), _i32(ml), _i32([step, 1]), 2, 1, fst, ms)
        st, _ = bso.advance(st, wp, t_idx, nf, ml, step, 0, 2, 1, fst.oracle)
        _same(dev.read(), st, step)
        t_idx = _reorder_t(t_idx, st["prev_ks"][step], K)
    assert st["err"][0] == (1 if ms < 6 else 0)
    assert (st["set_n"] <= ms).all()


def test_fst_fusion_every_branch_in_one_step():
    """hand-placed sets: a disambig state (4) emitting a token with arcs down the chain, the repeated label from state 2, the label
    with no arc (empty set, lm_scores -1e20), and finishes from the no-final state 5 (-inf) and from the chain"""
    K, B, V, step = 4, 2, 20, 3
    rng = np.random.default_rng(21)
    fst = Fst(V, 0.5, 0.2)
    arcs, _, _, _ = bso.fusion_lm(V)
    rep = [a[0] for i, a in enumerate(arcs[2][:-1]) if a[0] == arcs[2][i + 1][0]][0]
    st = random_state(B, K, V, step, rng, ms=8, fin_frac=0.0)
    po = step & 1
    st["set_n"][po] = 1
    st["set_state"][po, :, :, 0] = [[4, 2, 5, 3], [0, 4, 5, 3]]
    st["set_cost"][po, :, :, 0] = 0.5
    st["lm_scores"][:] = np.float32(-0.5)
    st["scores"][:] = [[0.0, -0.1, -0.2, -0.3], [0.0, -0.1, -0.2, -0.3]]
    x = np.full((B * K, V), -20.0, np.float32)
    for r, y in enumerate([12, rep - 1, 1, V - 1] + [V - 1, 1, 0, 0]):    # token 12 from state 4: three states, one reached twice
        x[r, y] = 10.0
    buf = torch.from_numpy(x).cuda()
    lse, wp = _word_probs(buf.data_ptr(), B * K, V, V, 1.0)
    nf = np.array([10, 10])
    t_idx = np.full(B * K, 9)                               # blank finishes
    dev = Dev(st)
    _advance(dev, buf.data_ptr(), lse, V, V, 1.0, _i32(t_idx), _i32(nf), _i32([10000, 10000]), _i32([step, 1]), 2, 1, fst, 8)
    want, _ = bso.advance(st, wp, t_idx, nf, [10000, 10000], step, 0, 2, 1, fst.oracle)
    got = dev.read()
    _same(got, want)
    assert (got["lm_scores"] == np.float32(-1e20)).any()
    assert np.isneginf(got["fin_score"]).any()
    assert (got["set_n"][po ^ 1] > 1).any()


# ------------------------------------------------------------------------------------------------ argument checks
def test_advance_argument_checks_launch_nothing():
    from pika_b200._lib import LmFst, PikaError, launch_count
    rng = np.random.default_rng(0)
    fst = Fst(20)
    n0 = launch_count()

    def call(K=4, V=20, ldv=20, null_lse=False, fs=None, ms=4):
        st = random_state(1, K, V, 1, rng, ms=4)
        dev = Dev(st)
        buf, addr, _ = _logits(K, V, max(ldv, V), 0, rng)
        lse = torch.zeros(K, device="cuda")
        if null_lse:
            lse = types.SimpleNamespace(data_ptr=lambda: None)
        z = _i32(np.zeros(K))
        with pytest.raises(PikaError):
            _advance(dev, addr, lse, ldv, V, 1.0, z, _i32([5]), _i32([100]), _i32([1, 1]), 1, 1, fs, ms)
        _same(dev.read(), st)

    call(K=3)
    call(K=32, V=40, ldv=40)
    call(K=8, V=6, ldv=6)
    call(ldv=19)
    call(null_lse=True)
    bad = LmFst()
    ctypes.memmove(ctypes.addressof(bad), ctypes.addressof(fst.struct), ctypes.sizeof(LmFst))
    bad.n_disambig = 5
    call(fs=types.SimpleNamespace(struct=bad, oracle=fst.oracle))
    call(fs=fst, ms=0)
    assert launch_count() == n0


def test_decoder_refuses_unsupported_widths_before_any_launch():
    from pika_b200._lib import PikaError, launch_count
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    m = _model(40)
    dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
    n0 = launch_count()
    for beam in (3, 32, 64):
        with pytest.raises(PikaError, match="beam sizes 1, 2, 4, 8, 16"):
            TransducerDecoder(m, 2, beam, n_best=1, blk=0, cuda=True, args=dargs)
    m2 = _model(12)
    dec = TransducerDecoder(m2, 2, 16, n_best=1, blk=0, cuda=True, args=dargs)
    with pytest.raises(PikaError, match="smaller than the beam"):
        dec.decode_batch(None, torch.tensor([10, 8]), max_len=[20, 20], enc_out=torch.zeros(2, 10, 1024, device="cuda"))
    assert launch_count() == n0


# ------------------------------------------------------------------------------------------------ the small step kernels
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_prepare(dtype):
    from pika_b200 import kernels as KK
    from pika_b200._lib import check, lib
    B, K, Tenc, H, E, ld_x, V, step = 3, 4, 7, 96, 20, 40, 11, 2
    rows = B * K
    g = torch.Generator().manual_seed(5)
    ny = torch.randint(-1, V, (step + 2, rows), generator=g, dtype=torch.int32)
    ny[step, :4] = torch.tensor([0, -1, 0, 3], dtype=torch.int32)
    t0 = torch.tensor([-1, 0, 6, 6, 2, 7, 5, 0, 3, 1, 6, 4], dtype=torch.int32)
    enc = torch.randn(B, Tenc, H, generator=g).to(dtype)
    emb = torch.randn(V, E, generator=g)
    t, enc_hid = t0.cuda(), torch.full((rows, H), 9.0, dtype=dtype, device="cuda")
    x = torch.full((rows, ld_x), 9.0, dtype=dtype, device="cuda")
    ny_d, ctx, enc_d, emb_d = ny.cuda(), _i32([step, 1]), enc.cuda(), emb.cuda()      # held: the kernel reads them after this line
    check(lib.pk_beam_prepare(ny_d.data_ptr(), ctx.data_ptr(), t.data_ptr(), enc_d.data_ptr(), KK._dt(enc), Tenc, H,
                              enc_hid.data_ptr(), emb_d.data_ptr(), E, x.data_ptr(), ld_x, K, 0, rows, _st()), "prepare")
    tok = ny[step].long()
    t_want = t0 + (tok == 0).int()
    assert t.cpu().tolist() == t_want.tolist()
    tc = t_want.clamp(0, Tenc - 1).long()
    assert torch.equal(enc_hid.cpu(), enc[torch.arange(rows) // K, tc])
    x_want = torch.zeros(rows, ld_x)
    real = tok > 0
    x_want[real, :E] = emb[tok[real]]
    assert torch.equal(x.cpu(), x_want.to(dtype))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_lstm_cell_and_gate(dtype):
    from pika_b200 import kernels as KK
    from pika_b200._lib import check, lib
    rows, H = 10, 200
    g = torch.Generator().manual_seed(6)
    gates = 2 * torch.randn(rows, 4 * H, generator=g)
    ny = torch.tensor([[0, 3, -1, 5, 0, 1, 7, -1, 2, 0]], dtype=torch.int32)
    h0, c0 = torch.randn(rows, H, generator=g).to(dtype), torch.randn(rows, H, generator=g)
    h, c = h0.cuda(), c0.cuda()
    gates_d, ny_d, ctx = gates.cuda(), ny.cuda(), _i32([0, 1])
    check(lib.pk_beam_lstm_cell(gates_d.data_ptr(), ny_d.data_ptr(), ctx.data_ptr(), 0, h.data_ptr(), KK._dt(h),
                                c.data_ptr(), rows, H, _st()), "lstm_cell")
    gd = gates.double()
    i, f, gg, o = gd[:, :H].sigmoid(), gd[:, H:2 * H].sigmoid(), gd[:, 2 * H:3 * H].tanh(), gd[:, 3 * H:].sigmoid()
    cw = f * c0.double() + i * gg
    hw = o * cw.tanh()
    m = ny[0] > 0
    assert torch.equal(h.cpu()[~m], h0[~m]) and torch.equal(c.cpu()[~m], c0[~m])
    tol = 1e-5 if dtype == torch.float32 else 8e-3
    assert (c.cpu()[m].double() - cw[m]).abs().max() < 1e-5
    assert (h.cpu()[m].double() - hw[m]).abs().max() < tol
    a = 3 * torch.randn(rows, 2 * H, generator=g)
    hj = torch.empty(rows, H, dtype=dtype, device="cuda")
    a_d = a.cuda()
    check(lib.pk_beam_gate(a_d.data_ptr(), hj.data_ptr(), KK._dt(hj), rows, H, _st()), "gate")
    ad = a.double()
    want = ad[:, :H].tanh() * ad[:, H:].sigmoid()
    assert (hj.cpu().double() - want).abs().max() < tol


@pytest.mark.parametrize("layers", [1, 2, 3])
def test_reorder(layers):
    from pika_b200._lib import PK_BF16, check, lib
    B, K, H, step = 3, 4, 72, 1
    rows = B * K
    g = torch.Generator().manual_seed(layers)
    pk = torch.stack([torch.randperm(K, generator=g) for _ in range(B)]).int()
    prev = torch.zeros(step + 1, rows, dtype=torch.int32)
    prev[step] = pk.reshape(-1)
    h, c = torch.randn(layers, rows, H, generator=g).bfloat16(), torch.randn(layers, rows, H, generator=g)
    t = torch.randint(0, 50, (rows,), generator=g, dtype=torch.int32)
    ho, co, to = torch.empty_like(h).cuda(), torch.empty_like(c).cuda(), torch.empty_like(t).cuda()
    prev_d, ctx, h_d, c_d, t_d = prev.cuda(), _i32([step, 1]), h.cuda(), c.cuda(), t.cuda()
    check(lib.pk_beam_reorder(prev_d.data_ptr(), ctx.data_ptr(), h_d.data_ptr(), c_d.data_ptr(), t_d.data_ptr(),
                              ho.data_ptr(), co.data_ptr(), to.data_ptr(), PK_BF16, K, H, layers, rows, _st()), "reorder")
    src = (torch.arange(rows) // K) * K + pk.reshape(-1).long()
    assert torch.equal(ho.cpu(), h[:, src]) and torch.equal(co.cpu(), c[:, src]) and torch.equal(to.cpu(), t[src])


def test_step_end_latch():
    from pika_b200._lib import check, lib
    nd = _i32([2])
    ctx = _i32([0, 1])
    for want in ([1, 1], [2, 1]):
        check(lib.pk_beam_step_end(ctx.data_ptr(), nd.data_ptr(), 10, _st()), "step_end")
        assert ctx.cpu().tolist() == want
    nd.zero_()
    check(lib.pk_beam_step_end(ctx.data_ptr(), nd.data_ptr(), 10, _st()), "step_end")
    assert ctx.cpu().tolist() == [3, 0]
    nd.fill_(5)                                           # dead stays dead
    check(lib.pk_beam_step_end(ctx.data_ptr(), nd.data_ptr(), 10, _st()), "step_end")
    assert ctx.cpu().tolist() == [3, 0]
    ctx = _i32([8, 1])
    check(lib.pk_beam_step_end(ctx.data_ptr(), nd.data_ptr(), 9, _st()), "step_end")
    assert ctx.cpu().tolist() == [9, 0]                   # max_steps


# ------------------------------------------------------------------------------------------------ transformer prediction net step
XF_STEP, XF_ROWS, XF_S1, XF_LAYERS = 40, 10, 302, 2
XF_VOCAB = 30


def _xf_setup(heads, dtype, ps, seed):
    """the state of pk_beam_xf_* at step XF_STEP: rows 0-5 compute position ps[row] (their earlier positions point at scattered pool
    entries of earlier steps); row 6 has a blank token, row 7 EOS, row 8 p = S1, and row 9's entry 1 + s*rows + 9 is n_entries: all
    four are inactive"""
    from pika_b200 import kernels as KK
    from pika_b200._lib import BeamXfState
    g = torch.Generator().manual_seed(seed)
    s, rows, S1 = XF_STEP, XF_ROWS, XF_S1
    D = 64 * heads
    n_entries = 1 + s * rows + 9
    ny = torch.randint(1, XF_VOCAB, (s + 2, rows), generator=g, dtype=torch.int32)
    ny[s, 6], ny[s, 7] = 0, -1
    hyp_len = torch.zeros(2, rows, dtype=torch.int32)
    hyp_len[s & 1] = torch.tensor(list(ps) + [5, 7, S1, 9], dtype=torch.int32)
    hyp_len[(s & 1) ^ 1] = torch.randint(0, S1, (rows,), generator=g, dtype=torch.int32)
    t = dict(next_ys=ny, hyp_len=hyp_len, ctx=torch.tensor([s, 1], dtype=torch.int32),
             hyp_tok=torch.randint(1, XF_VOCAB, (2, rows, S1), generator=g, dtype=torch.int32),
             slot=torch.randint(0, 1 + s * rows, (2, rows, S1), generator=g, dtype=torch.int32),
             pool=torch.randn(n_entries, XF_LAYERS, 3, D, generator=g).to(dtype))
    dv = {k: v.cuda() for k, v in t.items()}
    P = KK._P
    st = BeamXfState(P(dv["next_ys"]), P(dv["ctx"]), P(dv["hyp_tok"]), P(dv["hyp_len"]), P(dv["slot"]), P(dv["pool"]), n_entries, 0, rows, S1,
                     XF_LAYERS, D, KK._dt(dv["pool"]), 0)
    active = [r < len(ps) for r in range(rows)]
    return st, t, dv, active, g


XF_P = (0, 31, 32, 33, 64, 300)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("max_rel", [0, 1, 16])
@pytest.mark.parametrize("heads", [1, 8, 32])
def test_xf_attn_against_float64(heads, max_rel, dtype):
    """pk_beam_xf_attn at positions 0 to 300 (1 to 10 rounds of 32 keys) against a float64 softmax attention over the slot table;
    32 heads is a 1024-thread CTA.  The new K / V land in entry 1 + s*rows + row of the layer, nothing else of the pool changes, and
    inactive rows write zeros."""
    from pika_b200 import kernels as KK
    st, t, dv, active, g = _xf_setup(heads, dtype, XF_P, 100 * heads + max_rel)
    D, layer, s, par = 64 * heads, 1, XF_STEP, XF_STEP & 1
    qkv = torch.randn(XF_ROWS, 3 * D, generator=g).to(dtype)
    rel = torch.randn(2 * max_rel + 1, 64, generator=g) if max_rel else None
    qkv_d, rel_d = qkv.cuda(), (rel.cuda() if rel is not None else None)
    out = torch.full((XF_ROWS, D), 7.0, dtype=dtype, device="cuda")
    KK.beam_xf_attn(st, layer, qkv_d, heads, rel_d, out)
    got, pool = out.cpu().double(), dv["pool"].cpu()
    want_pool = t["pool"].clone()
    for r in range(XF_ROWS):
        if not active[r]:
            assert (got[r] == 0).all(), r
            continue
        e = 1 + s * XF_ROWS + r
        want_pool[e, layer, 0] = qkv[r, D:2 * D]
        want_pool[e, layer, 1] = qkv[r, 2 * D:]
        p = XF_P[r]
        ents = t["slot"][par, r, :p].long()
        kk = torch.cat([t["pool"][ents, layer, 0], qkv[r, D:2 * D][None]]).double().view(p + 1, heads, 64)
        vv = torch.cat([t["pool"][ents, layer, 1], qkv[r, 2 * D:][None]]).double().view(p + 1, heads, 64)
        q = qkv[r, :D].double().view(heads, 64) / 8.0
        sc = torch.einsum("hd,jhd->hj", q, kk)
        if max_rel:
            R = rel.double()[(torch.arange(p + 1) - p).clamp(min=-max_rel) + max_rel]
            sc = sc + torch.einsum("hd,jd->hj", q, R)
        pw = torch.softmax(sc, -1)
        o = torch.einsum("hj,jhd->hd", pw, vv)
        if max_rel:
            o = o + torch.einsum("hj,jd->hd", pw, R)
        o = o.reshape(D)
        tol = (2e-5 + 1e-5 * o.abs()) if dtype == torch.float32 else (1e-3 + 8e-3 * o.abs())
        assert ((got[r] - o).abs() <= tol).all(), (r, p, (got[r] - o).abs().max().item())
    assert torch.equal(pool, want_pool)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("layer", [0, 1])
def test_xf_taps(layer, dtype):
    """pk_beam_xf_taps: the causal conv's five taps of position p, zero before position 0 and past the C channels.  Layer 0 gathers
    embedding rows (blank at position 0) and records the row's entry in its slot table at p; layer 1 stores x_cur into the row's pool
    entry and reads the earlier positions through the slot table.  Inactive rows write zeros and touch neither pool nor slots."""
    from pika_b200 import kernels as KK
    ps = (0, 1, 3, 4, 5, 300)
    heads = 8
    st, t, dv, active, g = _xf_setup(heads, dtype, ps, 7 + layer)
    D, s, par = 64 * heads, XF_STEP, XF_STEP & 1
    E = 100
    emb = torch.randn(XF_VOCAB, E, generator=g)
    x_cur = torch.randn(XF_ROWS, D, generator=g).to(dtype)
    emb_d, x_d = emb.cuda(), x_cur.cuda()
    C, ldc = (E, 104) if layer == 0 else (D, D + 8)
    taps = torch.full((XF_ROWS, 5 * ldc), 7.0, dtype=dtype, device="cuda")
    KK.beam_xf_taps(st, layer, emb_d, x_d if layer else None, taps)
    got = taps.cpu().view(XF_ROWS, 5, ldc)
    want_pool, want_slot = t["pool"].clone(), t["slot"].clone()
    for r in range(XF_ROWS):
        if not active[r]:
            assert (got[r] == 0).all(), r
            continue
        p, e = ps[r], 1 + s * XF_ROWS + r
        want = torch.zeros(5, ldc, dtype=dtype)
        for k in range(5):
            j = p - 4 + k
            if j < 0:
                continue
            if layer == 0:
                want[k, :C] = emb[0 if j == 0 else int(t["hyp_tok"][par, r, j - 1])].to(dtype)
            else:
                want[k, :C] = x_cur[r] if j == p else t["pool"][int(t["slot"][par, r, j]), layer, 2]
        assert torch.equal(got[r], want), (r, p)
        if layer == 0:
            want_slot[par, r, p] = e
        else:
            want_pool[e, layer, 2] = x_cur[r]
    assert torch.equal(dv["pool"].cpu(), want_pool)
    assert torch.equal(dv["slot"].cpu(), want_slot)


# ------------------------------------------------------------------------------------------------ whole decodes at new widths
def _model(V, **reinit):
    from fixture_utils import decode_fixture_reinit
    from pika_b200.model.transducer import Net
    torch.manual_seed(777)
    args = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="transformer",
                                 embd_dim=100, padding_idx=V, dropout=0.2, dec_layers=2, enc_layers=9)
    m = Net(args, 240, V)
    decode_fixture_reinit(m, **reinit)
    return m.cuda().eval()


@pytest.mark.parametrize("beam,nbest,V,short", [(1, 1, 6000, False), (2, 2, 6000, False), (4, 2, 6500, False), (4, 2, 6000, True)],
                         ids=["K1", "K2", "K4-V6500", "K4-max_len"])
def test_decode_new_widths_against_oracle(beam, nbest, V, short):
    """fp32-class decodes from given encoder outputs (as the beam-16 fixture is run) against oracle.decode.decode_batch: tokens exact
    for n = 0 and wherever n-best neighbours are more than 5e-3 apart, scores 1e-3.  ``short``: max_len about half the frames, so
    hypotheses end on the length rule."""
    from make_inputs import DECODE_BIG_REINIT, decode_big_inputs
    from oracle import decode as od
    from pika_b200 import engine
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    B, Tp = 4, 40
    m = _model(V, **DECODE_BIG_REINIT)
    enc = torch.from_numpy(decode_big_inputs(606 + V + beam, B, Tp))
    tl = [40, 33, 27, 12]
    ml = [t // 2 for t in tl] if short else [t + 40 for t in tl]
    dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
    engine.set_precision("fp32")
    try:
        dec = TransducerDecoder(m, B, beam, n_best=nbest, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True,
                                args=dargs)
        ret, _ = dec.decode_batch(None, torch.tensor(tl), max_len=ml, enc_out=enc.cuda())
    finally:
        engine.set_precision("bf16")
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    try:
        ref = od.decode_batch(sd, enc, tl, beam, n_best=nbest, max_len=ml)
    finally:
        torch.set_num_threads(threads)
    for b in range(B):
        rs = ref["scores"][b]
        for n in range(nbest):
            sc = float(ret["scores"][b][n])
            assert abs(sc - rs[n]) < 1e-3 * abs(sc) + 1e-3, (b, n, sc, rs[n])
            gap = min([abs(rs[n] - rs[j]) for j in (n - 1, n + 1) if 0 <= j < nbest], default=1.0)
            if n == 0 or gap > 5e-3:
                hyp = [int(t) for t in ret["predictions"][b][n]]
                assert hyp == ref["predictions"][b][n], (b, n)
                if short:
                    assert len(hyp) == ml[b] - 1                 # ended on the length rule
