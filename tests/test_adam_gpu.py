"""Adam and BMUF-Adam on the GPU (pika_b200/csrc/optim.cu: pk_adam_clip, pk_bmuf_adam_update), the trainers built on them
(AdamClip, BmufAdamTrainer, BlockAdamTrainer) and the training entry point's ``--block_sync``.

* pk_adam_clip against torch.optim.Adam on CUDA (the foreach implementation) on the same tensors: every clip case, a
  fractional step count, n % 4 != 0, an unaligned buffer, the optional second output and a 91 M-element buffer.
* pk_bmuf_adam_update against the float32 restatement of the reference's update (the same roundings: bit-exact) and the
  float64 oracle (tests/adam_oracle.py), world 1 / 2 / 8.
* A transducer Net trained through AdamClip + BmufAdamTrainer for three blocks against the float64 oracle replaying the
  same gradients.
* The CLI with --block_sync bmuf_adam / block_adam, and the 2-GPU NCCL trajectory against the reference's own trainers
  (tests/golden/bmuf_adam_2rank.npz; skipped on a single-GPU machine)."""
import os
import sys

import numpy as np
import pytest
import torch

import adam_oracle as ao

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _rand(n, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(n) * scale).astype(np.float32)


def _ulps(a, b):
    """max |a - b| in ulps of max |b| (the vector's magnitude)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.spacing(F(np.abs(b).max())))


def _adam_vs_torch(n, clip, frac, offset=0, steps=3, lr=1e-2):
    from pika_b200 import kernels as K
    p0 = _rand(n, 1)
    # offset > 0: the buffers start 4 bytes past a 16-byte boundary, so the kernel runs its scalar path
    bufs = [torch.zeros(n + offset, device="cuda")[offset:] for _ in range(5)]
    p, g, m, v, out2 = bufs
    p.copy_(torch.from_numpy(p0))
    tp = torch.nn.Parameter(torch.from_numpy(p0.copy()).cuda())
    opt = torch.optim.Adam([tp], lr)                             # foreach on CUDA
    am = torch.zeros(1, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    step = 0.0
    worst = 0.0
    for it in range(steps):
        gh = _rand(n, 10 + it, 0.5 if it != 1 else 2.0)        # step 1 has the larger gradient (clip 3.0 becomes active there)
        g.copy_(torch.from_numpy(gh))
        tp.grad = torch.from_numpy(gh.copy()).cuda()
        if clip > 0:
            torch.nn.utils.clip_grad_norm_([tp], clip, norm_type=float("inf"))
            flag.zero_()
            K.absmax(g.clone() if offset else g, am, flag)     # pk_absmax reads float4: it needs a 16-byte aligned input
        opt.step()
        step = float(np.float32(step + 1))
        K.adam_clip(p, g, m, v, lr, (0.9, 0.999), 1e-8, step, clip, am, flag, p_out2=out2)
        if it == 0 and frac:
            opt.state[tp]["step"] += frac
            step = float(np.float32(np.float32(step) + np.float32(frac)))
        assert float(opt.state[tp]["step"]) == step
        tref = tp.detach().cpu().numpy()
        worst = max(worst, _ulps(p.cpu().numpy(), tref))
        np.testing.assert_allclose(m.cpu().numpy(), opt.state[tp]["exp_avg"].cpu().numpy(), rtol=0,
                                   atol=2 * np.spacing(F(opt.state[tp]["exp_avg"].abs().max().item())))
        np.testing.assert_allclose(v.cpu().numpy(), opt.state[tp]["exp_avg_sq"].cpu().numpy(), rtol=0,
                                   atol=2 * np.spacing(F(opt.state[tp]["exp_avg_sq"].abs().max().item())))
        assert torch.equal(out2, p)
    return worst


@pytest.mark.parametrize("n", [1, 7, 4096, (1 << 20) + 3])
@pytest.mark.parametrize("clip", [-1.0, 50.0, 3.0])
@pytest.mark.parametrize("frac", [0.0, 2.7])
def test_adam_clip_matches_torch_adam_cuda(n, clip, frac):
    """clip off / inactive / active (at step 1), an integer and a fractional step count: <= 2 ulp of |p|"""
    assert _adam_vs_torch(n, clip, frac) <= 2.0


def test_adam_clip_unaligned_buffers_take_the_scalar_path():
    assert _adam_vs_torch(4099, 3.0, 2.7, offset=1) <= 2.0


def test_adam_clip_91m_buffer():
    """the config-2 flat buffer size (91.4 M floats; not a multiple of 4 here), two steps"""
    assert _adam_vs_torch(91_400_003, 3.0, 0.0, steps=2) <= 2.0


def test_adam_clip_nan_propagates_like_torch():
    """clip_grad_norm_(inf) of a gradient holding one NaN: the coefficient is NaN and every parameter turns NaN"""
    from pika_b200 import kernels as K
    n = 1001
    gh = _rand(n, 3)
    gh[123] = np.nan
    g = torch.from_numpy(gh).cuda()
    p, m, v = torch.from_numpy(_rand(n, 4)).cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    am, flag = torch.zeros(1, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    K.absmax(g, am, flag)
    K.adam_clip(p, g, m, v, 1e-3, (0.9, 0.999), 1e-8, 1.0, 3.0, am, flag)
    tp = torch.nn.Parameter(torch.from_numpy(_rand(n, 4)).cuda())
    tp.grad = g.clone()
    torch.nn.utils.clip_grad_norm_([tp], 3.0, norm_type=float("inf"))
    torch.optim.Adam([tp], 1e-3).step()
    assert bool(torch.isnan(tp).all()) and bool(torch.isnan(p).all())


@pytest.mark.parametrize("n", [5, 4099, (1 << 20) + 4])
@pytest.mark.parametrize("world", [1, 2, 8])
def test_bmuf_adam_update_matches_oracle(n, world):
    """three consecutive syncs from the summed [delta; m; v]: bit-exact against the float32 restatement of the reference's
    tensor arithmetic; against float64, <= 2 ulp for the parameters and delta_prev and <= 4 ulp for the filtered moments (the
    reference's own float32 filter sits up to ~3 ulp from float64 there)"""
    from pika_b200 import kernels as K
    from test_bmuf_adam_gloo_cpu import NumpyOps
    bm, blr, tau, betas = 0.9, 1.0, 4, (0.9, 0.999)
    rng = np.random.default_rng(world * 7 + n)
    glob = rng.standard_normal(n).astype(F)
    dev = [torch.from_numpy(glob.copy()).cuda()] + [torch.zeros(n, device="cuda") for _ in range(4)]   # glob, local, dprev, m_g, v_g
    cpu = [t.cpu() for t in dev]
    rho = 0.0
    for it in range(3):
        ds, ms, vs = ((rng.standard_normal(n) * 0.01 * world).astype(F), (rng.standard_normal(n) * 0.01 * world).astype(F),
                      (rng.random(n) * 1e-4 * world).astype(F))
        msg_h = np.concatenate([ds, ms, vs])
        msg_d, msg_c = torch.from_numpy(msg_h).cuda(), torch.from_numpy(msg_h.copy())
        G, DP, MG, VG = (t.numpy().astype(np.float64) for t in (cpu[0], cpu[2], cpu[3], cpu[4]))
        G, DP, MG, VG, rho = ao.bmuf_adam_sync(G, DP, MG, VG, ds.astype(np.float64), ms.astype(np.float64), vs.astype(np.float64),
                                               world, bm, blr, betas, tau, rho)
        pw = (betas[0] ** tau, betas[0] ** (rho * bm), betas[1] ** tau, betas[1] ** (rho * bm))
        K.bmuf_adam_update(*dev, msg_d, world, bm, blr, *pw)
        NumpyOps.bmuf_adam_update(*cpu, msg_c, world, bm, blr, *pw)
        for a, b in zip(dev + [msg_d], cpu + [msg_c]):
            assert torch.equal(a.cpu(), b)
        assert torch.equal(dev[0], dev[1])
        assert torch.equal(msg_d[n:2 * n], dev[3]) and torch.equal(msg_d[2 * n:], dev[4])
        assert _ulps(dev[0].cpu(), G) <= 2 and _ulps(dev[2].cpu(), DP) <= 2
        assert _ulps(dev[3].cpu(), MG) <= 4 and _ulps(dev[4].cpu(), VG) <= 4


def _small_net():
    import types
    from pika_b200.model.transducer import Net
    d = np.load(os.path.join(ROOT, "tests", "golden", "model_small.npz"))
    V = int(d["V"])
    torch.manual_seed(777)
    margs = types.SimpleNamespace(rnn_size=512, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="rnn",
                                  embd_dim=100, padding_idx=V, dropout=0.0, dec_layers=1, enc_layers=2)     # 4.9 M parameters
    return Net(margs, 240, V).cuda().train(), d


def test_bmuf_adam_trains_a_transducer_net_like_the_oracle():
    """world 1: a small RNN-T Net (LSTM encoder) trained through AdamClip (clip 3.0) + BmufAdamTrainer, 2 local steps per block for three blocks,
    with the real kernels; the float64 oracle replays the same gradients.  Every sync re-stages the bf16 weight copies, so the
    losses of the next block come from the updated weights."""
    from pika_b200 import engine
    from pika_b200.trainer.bmuf import BmufAdamTrainer, SUCCESS
    from pika_b200.trainer.flat import AdamClip, FlatParams
    model, d = _small_net()
    flat = FlatParams(model)
    lr, bm, blr, tau, clip = 1e-4, 0.9, 1.0, 2, 3.0
    opt = AdamClip(flat, lr, max_norm=clip)
    tr = BmufAdamTrainer(0, 0, 1, model, bm, blr, tau, opt)
    glob = flat.data.double().cpu().numpy()
    p, m, v, step = glob.copy(), np.zeros_like(glob), np.zeros_like(glob), 0.0
    dprev, m_g, v_g, rho = np.zeros_like(glob), np.zeros_like(glob), np.zeros_like(glob), 0.0
    x, y = torch.from_numpy(d["x"]).cuda(), torch.from_numpy(d["y"]).long().cuda()
    tl, ul = torch.from_numpy(d["tlens"]).cuda(), torch.from_numpy(d["ulens"]).cuda()
    engine.set_precision("bf16")
    engine.set_dropout_enabled(False)
    losses = []
    try:
        for blk in range(3):
            for _ in range(tau):
                flat.zero_grad()
                costs = engine.transducer_loss(model, x, y, tl, ul, x_len=tl)
                costs.sum().backward()
                losses.append(float(costs.detach().sum()))
                g = flat.grad.cpu().numpy()
                opt.step()
                step = float(np.float32(step + 1))
                p, m, v = ao.adam_step(p, ao.clip_inf(g, clip).astype(np.float64), m, v, lr, (0.9, 0.999), 1e-8, step)
            assert tr.update_and_sync() == SUCCESS
            glob, dprev, m_g, v_g, rho = ao.bmuf_adam_sync(glob, dprev, m_g, v_g, glob - p, m, v, 1, bm, blr, (0.9, 0.999), tau, rho)
            p, m, v = glob.copy(), m_g.copy(), v_g.copy()
            step = float(np.float32(np.float32(step) + np.float32(rho * bm)))
            got = flat.data.cpu().numpy()
            assert opt.state[flat.params[0]]["step"] == step
            assert _ulps(got, glob) <= 4, (blk, _ulps(got, glob))
            # the moment filter cancels for some elements (values near 1e-11): bounded in ulps of the vector's magnitude
            assert _ulps(opt.exp_avg.cpu().numpy(), m_g) <= 4 and _ulps(opt.exp_avg_sq.cpu().numpy(), v_g) <= 4
            assert torch.equal(tr.param, flat.data)
    finally:
        engine.set_dropout_enabled(True)
    assert np.isfinite(losses).all() and losses[-1] < losses[0]


def _cli(tmp_path, block_sync, monkeypatch):
    from test_loader_cpu import make_dataset
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=8, shards=1, n_lo=14000, n_hi=22000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=0\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    out = tmp_path / "out"
    out.mkdir()
    log = tmp_path / "log.WORKER-ID"
    made = []

    def record(cls):
        class Rec(cls):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                made.append(self)
                self.seen = []

            def update_and_sync(self):
                rc = super().update_and_sync()
                opt = getattr(self, "optim", self)
                self.seen.append((opt.step_count, float(opt.exp_avg.abs().sum())))
                return rc
        return Rec
    monkeypatch.setattr(T, "BmufAdamTrainer", record(T.BmufAdamTrainer))
    monkeypatch.setattr(T, "BlockAdamTrainer", record(T.BlockAdamTrainer))
    # 8 utterances in batches of 4: 2 batches per epoch = 2 x sync_period, two epochs
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "transformer",
            "--decoder_type", "rnn", "--rnn_size", "1024", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60",
            "--padding_tgt", "60", "--dec_layers", "2", "--dropout", "0.0", "--brnn", "--model_lctx", "21", "--model_rctx", "21",
            "--model_stride", "4", "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--batch_size", "4",
            "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000", "--gain_range", "25,25",
            "--speed_rate", "1.0", "--grad_clip", "3.0", "--initial_lr", "1e-4", "--final_lr", "5e-5", "--num_epochs", "2",
            "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9", "--block_lr", "1e-3",
            "--block_sync", block_sync, "--seed", "777"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert "Training Finished" in text and len(losses) == 2 and np.isfinite(losses).all(), text
    assert len(made) == 1
    return made[0]


def test_cli_block_sync_bmuf_adam(tmp_path, monkeypatch):
    """one AdamClip for the whole run: the step count and moments carry over the epoch boundary"""
    tr = _cli(tmp_path, "bmuf_adam", monkeypatch)
    steps = [s for s, _ in tr.seen]
    assert len(steps) >= 4 and all(b > a for a, b in zip(steps, steps[1:]))
    assert all(mass > 0 for _, mass in tr.seen)
    assert tr.optim.lr == pytest.approx(np.exp(3 * np.log(0.5) / 4) * 1e-4)    # the schedule reached the optimiser via reset(lr)


def test_cli_block_sync_block_adam(tmp_path, monkeypatch):
    tr = _cli(tmp_path, "block_adam", monkeypatch)
    steps = [s for s, _ in tr.seen]
    assert steps == [float(i + 1) for i in range(len(steps))] and len(steps) >= 4
    assert all(mass > 0 for _, mass in tr.seen)


# ------------------------------------------------------------------------------------------------ 2 GPUs, NCCL
def _nccl_worker(which, rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    from make_golden_bmuf_adam import grad_vec, local_move
    from pika_b200.trainer.bmuf import BlockAdamTrainer, BmufAdamTrainer, SUCCESS
    from pika_b200.trainer.flat import AdamClip, FlatParams
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group(backend="nccl", init_method="env://", device_id=dev)
    torch.manual_seed(100 + rank)                      # same construction as make_golden_bmuf_adam.py
    model = torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.Linear(5, 3)).to(dev)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "bmuf_adam_2rank.npz"))
    ps = list(model.parameters())
    pvec = lambda ts: torch.nn.utils.parameters_to_vector(ts).detach().cpu().numpy()   # noqa: E731
    errs = []
    if which == "bmuf_adam":
        flat = FlatParams(model)
        opt = AdamClip(flat, float(gold["adam_lr"]))
        tr = BmufAdamTrainer(0, rank, world, model, float(gold["block_momentum"]), 1.0, int(gold["sync_period"]), opt)
        ok = np.array_equal(pvec(ps), gold["params"][0])
        for it in range(3):
            for k in range(int(gold["sync_period"])):
                g = grad_vec(it, k, rank, gold["params"].shape[1]).to(dev)
                off = 0
                for p in ps:
                    p.grad.copy_(g[off:off + p.numel()].view_as(p))
                    off += p.numel()
                opt.step()
            assert tr.update_and_sync() == SUCCESS
            errs.append((_ulps(pvec(ps), gold["params"][it + 1]), _ulps(pvec([opt.state[p]["exp_avg"] for p in ps]), gold["exp_avg"][it]),
                         _ulps(pvec([opt.state[p]["exp_avg_sq"] for p in ps]), gold["exp_avg_sq"][it])))
            ok &= max(errs[-1]) <= 2 and opt.state[ps[0]]["step"] == float(gold["step"][it])
    else:
        tr = BlockAdamTrainer(0, rank, world, model, float(gold["block_lr"]))
        ok = np.array_equal(pvec(ps), gold["block_adam_params"][0])
        for it in range(3):
            mv = local_move(it, rank, gold["block_adam_params"].shape[1]).to(dev)
            with torch.no_grad():
                off = 0
                for p in ps:
                    p.add_(mv[off:off + p.numel()].view_as(p))
                    off += p.numel()
            assert tr.update_and_sync() == SUCCESS
            errs.append(_ulps(pvec(ps), gold["block_adam_params"][it + 1]))
            ok &= errs[-1] <= 2
    q.put((rank, bool(ok), errs))
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("which", ["bmuf_adam", "block_adam"])
def test_nccl_two_gpus_match_reference_trajectory(which):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_nccl_worker, args=(which, r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(30)
    for r in res:
        assert r[1], r
