"""One-process-per-GPU plumbing for sharded sampling.

The reference's only multi-GPU mechanism is ``torch.nn.DataParallel`` around the network
(``models/utils.py:93``): every forward re-broadcasts all parameters (251 MB for the CIFAR-10
NCSN++) to every GPU and gathers outputs on ``cuda:0`` while the loop, the RNG and the
Langevin norms stay on one device.  Sample chains are independent, so the layout is one
process per GPU (``torchrun``), a full weight replica per rank broadcast **once** over
NCCL/NVLink, per-rank batches with per-rank seeds, **no collective inside the loop**, and one
final gather of the samples.

Batch coupling caveat: ``LangevinCorrector`` sets its step size from batch means of norms
(``sampling.py:276-278``).  Each rank's sub-batch is therefore *defined* as its own reference
batch: rank ``r`` equals the reference run with shape ``(B_r, ...)`` and seed ``seed + r``
``shard_batch`` gives the per-rank sizes; ``rank_seed`` the seed rule.
"""
import os

import torch
import torch.distributed as dist


def init_distributed(backend=None):
  """Initialise the default process group from the torchrun environment (no-op for 1 process).
  Returns ``(rank, world_size, local_rank)``."""
  world = int(os.environ.get('WORLD_SIZE', '1'))
  rank = int(os.environ.get('RANK', '0'))
  local = int(os.environ.get('LOCAL_RANK', '0'))
  if world > 1 and not dist.is_initialized():
    if backend is None:
      backend = 'nccl' if torch.cuda.is_available() else 'gloo'
    kw = {}
    if backend == 'nccl':
      torch.cuda.set_device(local)
      kw['device_id'] = torch.device('cuda', local)
    dist.init_process_group(backend, **kw)
  return rank, world, local


def shard_batch(total, world):
  """Sizes of the per-rank sub-batches of a ``total``-image request (remainder to the low ranks)."""
  base, rem = divmod(int(total), int(world))
  return [base + (1 if r < rem else 0) for r in range(world)]


def rank_seed(seed, rank):
  """Seed of rank ``rank``: the parity contract is 'rank r == reference run with seed + r'."""
  return int(seed) + int(rank)


def broadcast_parameters(model, src=0):
  """Make every rank's parameters and buffers equal to ``src``'s with one coalesced broadcast
  per dtype (NCCL over NVLink on GPUs, gloo in the CPU tests), then invalidate packed copies."""
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
    return model
  tensors = [p.data for p in model.parameters()] + [b.data for b in model.buffers()]
  by_dtype = {}
  for t in tensors:
    by_dtype.setdefault((t.dtype, t.device), []).append(t)
  for (_, _), group in by_dtype.items():
    flat = torch.cat([t.reshape(-1) for t in group])
    dist.broadcast(flat, src=src)
    off = 0
    for t in group:
      n = t.numel()
      t.copy_(flat[off:off + n].view_as(t))
      off += n
  if hasattr(model, 'invalidate_weights'):
    model.invalidate_weights()
  return model


def gather_samples(samples, dst=0):
  """Concatenate per-rank sample batches on ``dst`` (rank order).  Other ranks get ``None``.
  Per-rank batch sizes may differ (``shard_batch``)."""
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
    return samples
  world, rank = dist.get_world_size(), dist.get_rank()
  if samples.shape[0] == 0:
    # an empty shard may not know the image geometry: learn it from the other ranks
    geo = torch.tensor(list(samples.shape[1:]) + [0] * (3 - (samples.dim() - 1)), dtype=torch.long, device=samples.device)
    dist.all_reduce(geo, op=dist.ReduceOp.MAX)
    samples = samples.new_empty((0,) + tuple(int(v) for v in geo.tolist()))
  else:
    geo = torch.tensor(list(samples.shape[1:]), dtype=torch.long, device=samples.device)
    dist.all_reduce(geo, op=dist.ReduceOp.MAX)
  sizes = [torch.zeros(1, dtype=torch.long, device=samples.device) for _ in range(world)]
  dist.all_gather(sizes, torch.tensor([samples.shape[0]], dtype=torch.long, device=samples.device))
  sizes = [int(s.item()) for s in sizes]
  mx = max(sizes)
  pad = torch.zeros((mx,) + tuple(samples.shape[1:]), dtype=samples.dtype, device=samples.device)
  pad[:samples.shape[0]] = samples
  outs = [torch.empty_like(pad) for _ in range(world)]
  dist.all_gather(outs, pad)
  if rank != dst:
    return None
  return torch.cat([o[:n] for o, n in zip(outs, sizes)], dim=0)


def sharded_pc_sample(sampling_fn_factory, model, total_batch, seed):
  """Run a sampler on this rank's shard: ``sampling_fn_factory(batch)`` must return a
  ``sampling_fn(model)`` for that batch size (e.g. a ``get_sampling_fn`` closure).  Seeds the CPU and
  CUDA generators with ``rank_seed`` and returns ``(local_samples, nfe)``."""
  rank = dist.get_rank() if dist.is_initialized() else 0
  world = dist.get_world_size() if dist.is_initialized() else 1
  b = shard_batch(total_batch, world)[rank]
  torch.manual_seed(rank_seed(seed, rank))
  if torch.cuda.is_available():
    torch.cuda.manual_seed(rank_seed(seed, rank))
  if b == 0:
    # more ranks than images: contribute an empty batch so that gather_samples (a collective) still lines up
    try:
      probe = next(model.parameters())
      device = probe.device
    except (StopIteration, AttributeError):
      device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cpu')
    shape = getattr(sampling_fn_factory, 'sample_shape', None)
    tail = tuple(shape[1:]) if shape is not None else (0, 0, 0)
    return torch.empty((0,) + tail, dtype=torch.float32, device=device), 0
  return sampling_fn_factory(b)(model)
