#!/usr/bin/env python
"""Generate tests/golden/bmuf_adam_2rank.npz by EXECUTING THE REFERENCE's own trainer/bmuf.py:BmufAdamTrainer (with a real
torch.optim.Adam as its local optimiser) and trainer/bmuf.py:BlockAdamTrainer on 2 gloo ranks, imported from /root/reference
through tests/golden/ref_shim.py.  Environment repairs as make_golden.py:golden_bmuf: backend nccl -> gloo, ``.cuda(...)`` -> CPU.

Setup (the tests replay it):
  * model: torch.manual_seed(100 + rank); Sequential(Linear(7, 5), Linear(5, 3)) -- ranks start from different weights and
    rank 0's must win the initial broadcast;
  * BMUF-Adam: Adam(lr=ADAM_LR), block_momentum BM, block_lr 1.0, SYNC_PERIOD local Adam steps per block, three syncs; the
    gradient of local step k of block it on rank r is grad_vec(it, k, r) (one value per parameter, parameters_to_vector order);
  * block Adam: block_lr BLOCK_LR; before each of three syncs every rank moves its parameters by local_move(it, r).

Stored: the parameter vector after the broadcast and after every sync, for both trainers; for BMUF-Adam also the local
optimiser's exp_avg / exp_avg_sq (parameters_to_vector order) and state['step'] after every sync.

Run in the build container only:   python tests/golden/make_golden_bmuf_adam.py
The GPU box never runs this script.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ADAM_LR, BM, SYNC_PERIOD, BLOCK_LR = 1e-2, 0.9, 3, 1e-2


def grad_vec(it, k, rank, n):
    return 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(1000 * it + 10 * k + rank))


def local_move(it, rank, n):
    return 0.01 * torch.randn(n, generator=torch.Generator().manual_seed(500 + 7 * it + rank))


def _worker(which, rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    ref_shim.install()
    real_init = dist.init_process_group
    dist.init_process_group = lambda backend=None, **kw: real_init(backend="gloo", **kw)
    torch.Tensor.cuda = lambda self, *a, **k: self
    from trainer.bmuf import BlockAdamTrainer, BmufAdamTrainer, SUCCESS
    torch.manual_seed(100 + rank)
    model = torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.Linear(5, 3))
    vec = lambda ts: torch.nn.utils.parameters_to_vector(ts).detach().clone().numpy()   # noqa: E731
    out = dict(params=[])
    if which == "bmuf_adam":
        opt = torch.optim.Adam(model.parameters(), lr=ADAM_LR)
        tr = BmufAdamTrainer(0, rank, world, model, BM, 1.0, SYNC_PERIOD, opt)
        out.update(exp_avg=[], exp_avg_sq=[], step=[])
        out["params"].append(vec(model.parameters()))
        n = out["params"][0].size
        for it in range(3):
            for k in range(SYNC_PERIOD):
                g = grad_vec(it, k, rank, n)
                off = 0
                for p in model.parameters():
                    p.grad = g[off:off + p.numel()].view_as(p).clone()
                    off += p.numel()
                opt.step()
            assert tr.update_and_sync() == SUCCESS
            ps = list(model.parameters())
            out["params"].append(vec(ps))
            out["exp_avg"].append(vec([opt.state[p]["exp_avg"] for p in ps]))
            out["exp_avg_sq"].append(vec([opt.state[p]["exp_avg_sq"] for p in ps]))
            steps = {float(opt.state[p]["step"]) for p in ps}
            assert len(steps) == 1
            out["step"].append(steps.pop())
    else:
        tr = BlockAdamTrainer(0, rank, world, model, BLOCK_LR)
        out["params"].append(vec(model.parameters()))
        n = out["params"][0].size
        for it in range(3):
            with torch.no_grad():
                torch.nn.utils.vector_to_parameters(torch.from_numpy(vec(model.parameters())) + local_move(it, rank, n),
                                                    model.parameters())
            assert tr.update_and_sync() == SUCCESS
            out["params"].append(vec(model.parameters()))
    q.put((rank, {k: np.array(v) for k, v in out.items()}))
    dist.destroy_process_group()


def run(which, port):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(which, r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(30)
    # the broadcast leaves every rank with the same parameters, moments and step after each sync
    for k in res[0][1]:
        assert np.array_equal(res[0][1][k], res[1][1][k]), (which, k)
    return res[0][1]


def main():
    a = run("bmuf_adam", 29300 + (os.getpid() % 500))
    b = run("block_adam", 29900 + (os.getpid() % 500))
    np.savez_compressed(os.path.join(HERE, "bmuf_adam_2rank.npz"), params=a["params"], exp_avg=a["exp_avg"],
                        exp_avg_sq=a["exp_avg_sq"], step=a["step"], block_adam_params=b["params"],
                        adam_lr=ADAM_LR, block_momentum=BM, sync_period=SYNC_PERIOD, block_lr=BLOCK_LR)
    print("bmuf_adam: params", a["params"].shape, "steps", a["step"], "| block_adam: params", b["params"].shape)


if __name__ == "__main__":
    main()
