"""BMUF (block-wise model update filtering) -- drop-in for trainer/bmuf.py (reference): BmufTrainer, BlockAdamTrainer and
BmufAdamTrainer.

Same constructor and methods (``update_and_sync() -> SUCCESS|STOP``, ``sum_reduce``, ``broadcast``).
GPU mapping: the reference's ``reduce(delta -> rank 0)`` / rank-0 update / ``broadcast(param)``
(trainer/bmuf.py:83-98) is one NCCL all-reduce over NVLink of the flat delta followed by
the identical fused block-momentum update on every rank (``delta_prev`` is replicated instead of living
on rank 0 only); parameters are views of the flat buffer, so there are no flatten / un-flatten copies.
The NaN guard is made collective (the reference lets only the ranks that see NaN return early and the
others hang in ``broadcast`` -- SURVEY.md section 5).
"""
import torch
import torch.distributed as dist

from .. import engine
from .. import kernels as K
from .flat import AdamClip, FlatParams, f32

SUCCESS = 1
STOP = 0


class _Collectives:
    """the trainer-facing collective helpers every block trainer offers"""

    def broadcast(self, tensor):
        """broadcast interface for trainer"""
        if self.world_size > 1:
            dist.broadcast(tensor=tensor, src=self.master_node)

    def sum_reduce(self, tensor):
        """sumreduce interface for trainer (result valid on the master node, as in the reference)"""
        if self.world_size > 1:
            dist.reduce(tensor=tensor, dst=self.master_node)


class BmufTrainer(_Collectives):
    """
    Args (as in the reference):
        master_node (int), rank (int), world_size (int), model (nn.Module),
        block_momentum (float), block_lr (float)
    Extra keyword: ``flat`` -- an existing FlatParams of ``model`` (created when omitted);
    ``backend`` -- "nccl" (default, as hard-coded in the reference) or "gloo" for CPU-side tests.
    """

    def __init__(self, master_node, rank, world_size, model, block_momentum, block_lr, flat=None, backend="nccl", ops=None):
        # ``ops``: object with bmuf_delta / bmuf_update / absmax; defaults to the CUDA kernels.  The CPU-side
        # gloo test injects the numpy oracle here to exercise the collective protocol without a GPU.
        self.ops = ops if ops is not None else K
        self.master_node, self.rank, self.world_size = master_node, rank, world_size
        self.model, self.block_momentum, self.block_lr = model, block_momentum, block_lr
        if world_size > 1 and not dist.is_initialized():
            dist.init_process_group(backend=backend, init_method="env://")
        self.flat = flat if flat is not None else FlatParams(model)
        self.param = self.flat.data.clone()              # the global (block) model
        if world_size > 1:
            dist.broadcast(tensor=self.param, src=master_node)
            self.flat.data.copy_(self.param)
            engine.invalidate_weights()
        self.delta_prev = torch.zeros_like(self.param)
        self.delta = torch.zeros_like(self.param)
        if world_size > 1:
            # the first all-reduce of a communicator sets up its channels / buffers for this message size and costs far more than every
            # later block sync: pay that at construction, next to the parameter broadcast, not in the first block
            dist.all_reduce(self.delta, op=dist.ReduceOp.SUM)
        self.health = torch.zeros(2, dtype=torch.float32, device=self.param.device)   # [absmax, unused]
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=self.param.device)

    def update_and_sync(self):
        """one block sync: returns SUCCESS if numerics are healthy on every rank, STOP otherwise"""
        self.ops.bmuf_delta(self.param, self.flat.data, self.delta)
        if self.world_size > 1:
            dist.all_reduce(self.delta, op=dist.ReduceOp.SUM)
        self.nan_flag.zero_()
        self.ops.absmax(self.delta, self.health[:1], self.nan_flag)     # NaNs propagate through the sum: every rank sees them
        if int(self.nan_flag.item()) != 0:
            return STOP
        self.ops.bmuf_update(self.param, self.flat.data, self.delta_prev, self.delta, self.world_size, self.block_momentum, self.block_lr)
        engine.invalidate_weights()
        return SUCCESS


class _AdamBlockTrainer(_Collectives):
    """what the two Adam block trainers share: process group, flat parameters, broadcast of rank 0's weights and the
    collective NaN check"""

    def _setup(self, master_node, rank, world_size, model, flat, backend, ops):
        self.ops = ops if ops is not None else K
        self.master_node, self.rank, self.world_size, self.model = master_node, rank, world_size, model
        if world_size > 1 and not dist.is_initialized():
            dist.init_process_group(backend=backend, init_method="env://")
        self.flat = flat if flat is not None else FlatParams(model)
        self.param = self.flat.data.clone()              # the global (block) model
        if world_size > 1:
            dist.broadcast(tensor=self.param, src=master_node)
            self.flat.data.copy_(self.param)
            engine.invalidate_weights()
        self.health = torch.zeros(1, dtype=torch.float32, device=self.param.device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=self.param.device)

    def _all_reduce_is_finite(self, vec):
        """sum ``vec`` over ranks in place; False when it holds a NaN (NaNs propagate through the sum: every rank sees them)"""
        if self.world_size > 1:
            dist.all_reduce(vec, op=dist.ReduceOp.SUM)
        self.nan_flag.zero_()
        self.ops.absmax(vec, self.health, self.nan_flag)
        return int(self.nan_flag.item()) == 0


class BlockAdamTrainer(_AdamBlockTrainer):
    """Drop-in for trainer/bmuf.py:BlockAdamTrainer: Adam at ``block_lr`` applied to the block delta SUMMED over ranks (the
    reference does not divide it by the world size, :161), with the Adam state replicated on every rank instead of living on the
    master.  The update writes the global vector and the model's flat buffer in one pass (pk_adam_clip's second output).
    Extra keywords as BmufTrainer's (``flat``, ``backend``, ``ops``)."""

    def __init__(self, master_node, rank, world_size, model, block_lr, flat=None, backend="nccl", ops=None):
        self._setup(master_node, rank, world_size, model, flat, backend, ops)
        self.block_lr = block_lr
        self.betas, self.eps = (0.9, 0.999), 1e-8       # torch.optim.Adam([param], block_lr, weight_decay=0.0) (:142)
        self.step_count = 0.0
        self.exp_avg = torch.zeros_like(self.param)
        self.exp_avg_sq = torch.zeros_like(self.param)
        self.delta = torch.zeros_like(self.param)
        if world_size > 1:
            # pay the communicator's first-call setup at this message size now, not in the first block (as BmufTrainer)
            dist.all_reduce(self.delta, op=dist.ReduceOp.SUM)

    def update_and_sync(self):
        """one block sync: returns SUCCESS if numerics are healthy on every rank, STOP otherwise"""
        self.ops.bmuf_delta(self.param, self.flat.data, self.delta)
        if not self._all_reduce_is_finite(self.delta):
            return STOP
        self.step_count = f32(self.step_count + 1)
        self.ops.adam_clip(self.param, self.delta, self.exp_avg, self.exp_avg_sq, self.block_lr, self.betas, self.eps,
                           self.step_count, p_out2=self.flat.data)
        engine.invalidate_weights()
        return SUCCESS

    def get_block_lr(self):
        """get current learning rate"""
        return self.block_lr

    def set_block_lr(self, value):
        """set a new learning rate"""
        self.block_lr = value


class BmufAdamTrainer(_AdamBlockTrainer):
    """Drop-in for trainer/bmuf.py:BmufAdamTrainer (BMUF-Adam, Chen et al. 2020): each rank runs a local Adam (``optim``, an
    ``AdamClip`` over the same FlatParams); at every block sync the block delta AND the local Adam moments are summed over
    ranks, the global model takes a block-momentum step, and the averaged moments are filtered into the next block's moments.

    GPU mapping: the reference's cat of [delta; exp_avg; exp_avg_sq] (:254-267) / reduce to the master / master update /
    broadcast / per-parameter copies (:298-321) become one NCCL all-reduce of a 3n message and one fused update replicated on
    every rank.  The optimiser's moment buffers ARE slots 1 and 2 of that message, so nothing is gathered; they are reduced in
    place, which is safe because the sync overwrites them anyway (:314-319).  Extra keywords as BmufTrainer's."""

    def __init__(self, master_node, rank, world_size, model, block_momentum, block_lr, sync_period, optim, flat=None,
                 backend="nccl", ops=None):
        if not isinstance(optim, AdamClip):
            raise TypeError("BmufAdamTrainer needs a pika_b200.trainer.flat.AdamClip optimiser (got %s): the local Adam step, "
                            "like every update on this path, runs as a CUDA kernel over the flat buffers"
                            % type(optim).__name__)
        if flat is not None and optim.flat is not flat:
            raise ValueError("BmufAdamTrainer: optim and flat must share one FlatParams")
        self._setup(master_node, rank, world_size, model, optim.flat, backend, ops)
        self.block_momentum, self.block_lr, self.sync_period, self.optim = block_momentum, block_lr, sync_period, optim
        self.rho = 0.0
        self.betas = tuple(optim.betas)
        n = self.param.numel()
        self.delta_prev = torch.zeros_like(self.param)
        self.exp_avg = torch.zeros_like(self.param)     # the filtered global moments (master-only in the reference, :241-243)
        self.exp_avg_sq = torch.zeros_like(self.param)
        self.msg = torch.zeros(3 * n, dtype=torch.float32, device=self.param.device)     # [delta; local exp_avg; local exp_avg_sq]
        optim.place_moments(self.msg[n:2 * n], self.msg[2 * n:])
        # the reference skips parameters whose .grad is None when it gathers the moments (:260, :308); every FlatParams
        # parameter has a gradient view into the flat gradient buffer, so here every slot takes part
        if world_size > 1:
            # warm-up at the 3n message size (see BmufTrainer); reduces nothing but zeros: the local moments start at zero
            # and the delta slot is rewritten at every sync
            dist.all_reduce(torch.zeros_like(self.msg), op=dist.ReduceOp.SUM)

    def update_and_sync(self):
        """one block sync: returns SUCCESS if numerics are healthy on every rank, STOP otherwise (rho is then unchanged)"""
        n = self.param.numel()
        self.ops.bmuf_delta(self.param, self.flat.data, self.msg[:n])
        if not self._all_reduce_is_finite(self.msg):
            return STOP
        bm, tau = self.block_momentum, self.sync_period
        self.rho = bm * self.rho + tau
        b1, b2 = self.betas
        self.ops.bmuf_adam_update(self.param, self.flat.data, self.delta_prev, self.exp_avg, self.exp_avg_sq, self.msg,
                                  self.world_size, bm, self.block_lr, b1 ** tau, b1 ** (self.rho * bm), b2 ** tau, b2 ** (self.rho * bm))
        # state['step'] += rho * block_momentum (:311), in the float32 arithmetic of torch's step tensor
        self.optim.step_count = f32(self.optim.step_count + f32(self.rho * bm))
        engine.invalidate_weights()
        return SUCCESS
