"""BmufAdamTrainer and BlockAdamTrainer across 2 ranks on CPU (gloo): the collective protocol (initial broadcast, one
all-reduce of the 3n message [delta; exp_avg; exp_avg_sq], replicated update, collective NaN stop, step bookkeeping, the
optimiser's moments aliasing the message) and the trajectories of the reference's own trainers run on 2 gloo ranks
(tests/golden/bmuf_adam_2rank.npz, make_golden_bmuf_adam.py).  The element-wise kernels are CUDA-only, so this host-logic
test injects float32 numpy implementations of the ops through ``ops=``."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "bmuf_adam_2rank.npz")
F = np.float32


def _fma(a, b, c):
    """float32 a * b + c with one rounding (exact product in float64), as torch's CPU kernels fuse it"""
    return (np.float64(a) * np.asarray(b, np.float64) + c).astype(F)


class NumpyOps:
    """float32 with the roundings of torch's CPU tensor ops (the reference runs torch on the CPU): one per op, except the
    multiply-adds that torch's CPU lerp_ and addcmul_ fuse"""

    @staticmethod
    def bmuf_delta(glob, local, delta):
        delta.copy_(glob - local)

    @staticmethod
    def absmax(x, out, nan_flag):
        out[0] = x.abs().max() if not torch.isnan(x).any() else float("nan")
        if torch.isnan(x).any():
            nan_flag[0] = 1

    @staticmethod
    def adam_clip(p, g, m, v, lr, betas, eps, step, max_norm=-1.0, absmax_t=None, nan_flag=None, p_out2=None):
        b1, b2 = betas
        P, G, M, V = (t.numpy() for t in (p, g, m, v))
        if max_norm > 0:
            coef = F(max_norm) / (F(np.abs(G).max()) + F(1e-6))
            G = G * min(coef, F(1.0))
        M[:] = _fma(F(1 - b1), G - M, M)
        V[:] = _fma(F(1 - b2) * G, G, V * F(b2))
        den = np.sqrt(V) / F((1 - b2 ** step) ** 0.5) + F(eps)
        P[:] = P + F(-(lr / (1 - b1 ** step))) * (M / den)
        if p_out2 is not None:
            p_out2.copy_(p)

    @staticmethod
    def bmuf_adam_update(glob, local, dprev, m_g, v_g, msg, world, bm, blr, b1t, b1r, b2t, b2r):
        n = glob.numel()
        vec = msg.numpy() / F(world)
        Gl, DP, MG, VG = (t.numpy() for t in (glob, dprev, m_g, v_g))
        DP[:] = F(bm) * DP + F(blr * (1 - bm)) * vec[:n]
        Gl[:] = Gl - F(1 + bm) * DP
        MG[:] = (F(b1t * (b1r - 1)) * MG + F(1 - b1t * b1r) * vec[n:2 * n]) / F(1 - b1t)
        VG[:] = (F(b2t * (b2r - 1)) * VG + F(1 - b2t * b2r) * vec[2 * n:]) / F(1 - b2t)
        local.copy_(glob)
        msg[n:2 * n].copy_(m_g)
        msg[2 * n:].copy_(v_g)


def _pvec(ts):
    return torch.nn.utils.parameters_to_vector(ts).detach().numpy().copy()


def _ulp_close(a, b, k=2):
    """|a - b| <= k ulp of the vector's magnitude"""
    return bool(np.abs(a - b).max() <= k * np.spacing(F(np.abs(b).max())))


def _init(rank, world, port):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.manual_seed(100 + rank)                      # ranks start from DIFFERENT weights: rank 0's must win
    return torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.Linear(5, 3))


def _gather(t):
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t.clone())
    return out


def bmuf_adam_worker(rank, world, port, q):
    model = _init(rank, world, port)
    import adam_oracle as ao
    from make_golden_bmuf_adam import grad_vec
    from pika_b200.trainer.bmuf import BmufAdamTrainer, SUCCESS, STOP
    from pika_b200.trainer.flat import AdamClip, FlatParams, f32
    gold = np.load(GOLD)
    lr, bm, tau = float(gold["adam_lr"]), float(gold["block_momentum"]), int(gold["sync_period"])
    res = {}
    # a torch optimiser is refused: nothing on this path computes in torch
    try:
        BmufAdamTrainer(0, rank, world, torch.nn.Linear(2, 2), bm, 1.0, tau, torch.optim.Adam(torch.nn.Linear(2, 2).parameters()))
        res["type_error"] = False
    except TypeError:
        res["type_error"] = True
    flat = FlatParams(model)
    opt = AdamClip(flat, lr, ops=NumpyOps)
    tr = BmufAdamTrainer(0, rank, world, model, bm, 1.0, tau, opt, backend="gloo", ops=NumpyOps)
    ps = list(model.parameters())
    n = flat.numel
    res["broadcast"] = np.array_equal(_pvec(ps), gold["params"][0]) and all(torch.equal(x, tr.param) for x in _gather(tr.param))
    # state[p]['exp_avg'] / ['exp_avg_sq'] are views of the message's moment slots, which the optimiser updates in place
    base, es = tr.msg.data_ptr(), tr.msg.element_size()
    res["alias"] = all(opt.state[p]["exp_avg"].data_ptr() == base + es * (n + o) and
                       opt.state[p]["exp_avg_sq"].data_ptr() == base + es * (2 * n + o) for p, o in zip(ps, flat.offsets))
    glob, dprev, m_g, v_g, rho = (tr.param.numpy().astype(np.float64), np.zeros(n), np.zeros(n), np.zeros(n), 0.0)
    ok_sum = ok_oracle = ok_gold = ok_step = True
    for it in range(3):
        for k in range(tau):
            g = grad_vec(it, k, rank, int(gold["params"].shape[1]))
            off = 0
            for p in ps:
                p.grad.copy_(g[off:off + p.numel()].view_as(p))
                off += p.numel()
            opt.step()
        res["alias"] &= torch.equal(opt.state[ps[0]]["exp_avg"].reshape(-1), tr.msg[n:n + ps[0].numel()])
        res["alias"] &= bool(tr.msg[n:].abs().max() > 0)
        locals_ = _gather(flat.data)
        ms, vs = _gather(opt.exp_avg), _gather(opt.exp_avg_sq)
        step_before = opt.state[ps[0]]["step"]
        gp = tr.param.clone()
        assert tr.update_and_sync() == SUCCESS
        # slot 0 of the message holds the delta summed over the ranks (the 3n all-reduce)
        expect = sum((gp - l_).numpy().astype(np.float64) for l_ in locals_)
        ok_sum &= np.allclose(tr.msg[:n].numpy(), expect, rtol=0, atol=1e-6)
        glob, dprev, m_g, v_g, rho = ao.bmuf_adam_sync(glob, dprev, m_g, v_g, expect, sum(x.numpy().astype(np.float64) for x in ms),
                                                       sum(x.numpy().astype(np.float64) for x in vs), world, bm, 1.0,
                                                       (0.9, 0.999), tau, rho)
        ok_oracle &= (tr.rho == rho and np.allclose(tr.param.numpy(), glob, rtol=0, atol=1e-6) and torch.equal(tr.param, flat.data)
                      and np.allclose(opt.exp_avg.numpy(), m_g, rtol=1e-5, atol=1e-9)
                      and np.allclose(opt.exp_avg_sq.numpy(), v_g, rtol=1e-5, atol=1e-12))
        ok_step &= opt.state[ps[-1]]["step"] == f32(step_before + f32(rho * bm)) == float(gold["step"][it])
        ok_gold &= (_ulp_close(_pvec(ps), gold["params"][it + 1]) and
                    _ulp_close(_pvec([opt.state[p]["exp_avg"] for p in ps]), gold["exp_avg"][it]) and
                    _ulp_close(_pvec([opt.state[p]["exp_avg_sq"] for p in ps]), gold["exp_avg_sq"][it]))
    res.update(sum=ok_sum, oracle=ok_oracle, step=ok_step, gold=ok_gold)
    # collective NaN stop: only rank 1 diverges, EVERY rank returns STOP, and rho is not advanced
    rho_before = tr.rho
    if rank == 1:
        with torch.no_grad():
            flat.data[3] = float("nan")
    res["stop"] = tr.update_and_sync() == STOP and tr.rho == rho_before
    t = torch.tensor([float(rank + 1), 10.0])
    tr.sum_reduce(t)
    tr.broadcast(t)
    res["helpers"] = abs(t[0].item() - sum(range(1, world + 1))) < 1e-6
    q.put((rank, res))
    dist.destroy_process_group()


def block_adam_worker(rank, world, port, q):
    model = _init(rank, world, port)
    import adam_oracle as ao
    from make_golden_bmuf_adam import local_move
    from pika_b200.trainer.bmuf import BlockAdamTrainer, SUCCESS, STOP
    gold = np.load(GOLD)
    blr = float(gold["block_lr"])
    tr = BlockAdamTrainer(0, rank, world, model, blr, backend="gloo", ops=NumpyOps)
    ps = list(model.parameters())
    n = tr.flat.numel
    res = dict(broadcast=np.array_equal(_pvec(ps), gold["block_adam_params"][0]), lr=tr.get_block_lr() == blr)
    glob, m, v, step = tr.param.numpy().astype(np.float64), np.zeros(n), np.zeros(n), 0.0
    ok_sum = ok_oracle = ok_gold = True
    for it in range(3):
        mv = local_move(it, rank, int(gold["block_adam_params"].shape[1]))
        with torch.no_grad():
            off = 0
            for p in ps:
                p.add_(mv[off:off + p.numel()].view_as(p))
                off += p.numel()
        locals_ = _gather(tr.flat.data)
        gp = tr.param.clone()
        assert tr.update_and_sync() == SUCCESS
        expect = sum((gp - l_).numpy().astype(np.float64) for l_ in locals_)
        ok_sum &= np.allclose(tr.delta.numpy(), expect, rtol=0, atol=1e-6)     # summed, NOT averaged (:161)
        glob, m, v, step = ao.block_adam_sync(glob, m, v, step, expect, blr)
        ok_oracle &= np.allclose(tr.param.numpy(), glob, rtol=0, atol=1e-6) and torch.equal(tr.param, tr.flat.data)
        ok_gold &= _ulp_close(_pvec(ps), gold["block_adam_params"][it + 1])
    res.update(sum=ok_sum, oracle=ok_oracle, gold=ok_gold, step=tr.step_count == 3.0)
    tr.set_block_lr(0.5 * blr)
    res["lr"] &= tr.get_block_lr() == 0.5 * blr
    if rank == 1:
        with torch.no_grad():
            tr.flat.data[3] = float("nan")
    res["stop"] = tr.update_and_sync() == STOP and tr.step_count == 3.0
    q.put((rank, res))
    dist.destroy_process_group()


def _run(target, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=100) for _ in procs]
    for p in procs:
        p.join(30)
    for rank, r in res:
        assert all(r.values()), (rank, r)


@pytest.mark.timeout(120)
def test_bmuf_adam_two_ranks_gloo():
    _run(bmuf_adam_worker, 33500 + (os.getpid() % 2000))


@pytest.mark.timeout(120)
def test_block_adam_two_ranks_gloo():
    _run(block_adam_worker, 35500 + (os.getpid() % 2000))
