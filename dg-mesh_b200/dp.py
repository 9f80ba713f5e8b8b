"""Data parallelism over training frames (SURVEY.md 8(e)) -- new in this implementation: the reference
is single-process (dgmesh/train.py renders one frame per iteration on cuda:0).

A frame's forward/backward depends only on the replicated parameters, its camera and its time, so
frame k of a batch goes to rank k % world and the only data-path exchange is ONE all-reduce (NCCL over
NVLink on a multi-GPU H100 node, gloo in the CPU tests) of a single flat fp32 buffer holding every gradient:
canonical-Gaussian parameters followed by the MLP parameters.  Batch of one frame per step -> no
collective at all.  Densification statistics need the same reduction so all ranks prune identically
(gaussian_model_dpsr_dynamic_anchor.py:679-682)."""
import os
import sys

import torch
import torch.distributed as dist

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)


def shard_frames(n_frames, rank, world):
    """Frame indices of this rank (round-robin, like the one-frame-per-GPU layout of an 8-GPU node)."""
    return [k for k in range(n_frames) if k % world == rank]


class FlatGrad:
    """Gradients of `params` as views of ONE flat buffer, so the exchange is a single collective.

    The views are installed as `p.grad`.  A training loop may break that aliasing -- the reference's
    `optimizer.zero_grad(set_to_none=True)` (dgmesh/train.py:525-530) drops the views, and
    densification replaces the Parameter objects altogether -- so `allreduce()` verifies every binding
    first: a detached `p.grad` is copied into its slice and re-bound (correct result, one extra copy), a
    missing one counts as zero, and a parameter list whose shapes changed raises.  After densify / prune
    call `rebuild(new_params)`; use `zero()` (or `zero_grad(set_to_none=False)`) to keep the fast path."""

    def __init__(self, params):
        self.rebuild(params)

    def rebuild(self, params):
        """(Re)create the flat buffer for a new parameter list (after densification / pruning)."""
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("FlatGrad: no parameter requires grad")
        dev, dt = self.params[0].device, torch.float32
        self.flat = torch.zeros(sum(p.numel() for p in self.params), device=dev, dtype=dt)
        self.offsets, self.shapes, off = [], [], 0
        for p in self.params:
            self.offsets.append(off)
            self.shapes.append(tuple(p.shape))
            off += p.numel()
        self._bind(copy=False)

    def _slice(self, i):
        if tuple(self.params[i].shape) != self.shapes[i]:
            raise RuntimeError("FlatGrad: a parameter changed shape; call rebuild(params) after densify / prune")
        n = 1
        for d in self.shapes[i]:
            n *= d
        return self.flat[self.offsets[i]:self.offsets[i] + n].view(self.shapes[i])

    def _bind(self, copy):
        """Make every p.grad a view of the flat buffer; returns how many had to be re-bound."""
        rebound = 0
        for i, p in enumerate(self.params):
            v = self._slice(i)
            g = p.grad
            if g is not None and g.data_ptr() == v.data_ptr() and g.shape == v.shape:
                continue
            if copy:
                if g is None:
                    v.zero_()          # no gradient this step (e.g. zero_grad(set_to_none=True) and unused)
                else:
                    v.copy_(g)
            p.grad = v
            rebound += 1
        return rebound

    def zero(self):
        self.flat.zero_()

    def allreduce(self, average=True, group=None):
        """Sum (or mean) of the gradients over the ranks; no-op for a single process."""
        self._bind(copy=True)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
            if average:
                self.flat.div_(dist.get_world_size(group))
        return self.flat


class NvlsFlatGrad(FlatGrad):
    """`FlatGrad` whose buffer lives in symmetric memory behind an NVSwitch MULTICAST mapping, all-reduced by
    this library's own kernel (csrc/nvls.cu: the switch performs the reduction -- `multimem.ld_reduce` of this
    rank's slice, `multimem.st` of the result to every replica; one launch, two flag barriers) instead of
    ncclAllReduce.  At the sizes of this path (24-60 MB) the NCCL call is latency-bound; see DESIGN.md 5.

    Needs a NCCL process group (for the rendezvous only) on GPUs joined by NVSwitch; raises if the platform has
    no multicast support (use `FlatGrad` there).  torch's symmetric-memory allocator is plumbing: it provides
    the memory, the multicast address and the signal pads; the collective itself is ours."""

    BLOCKS = 264     # two per SM (H100: 132): enough multimem requests in flight to fill the links
    PAD_SKIP = 128

    def __init__(self, params, group=None):
        self.group = group
        self._epoch = 1
        self._handle = None
        super().__init__(params)

    def rebuild(self, params):
        import torch.distributed._symmetric_memory as symm_mem
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("FlatGrad: no parameter requires grad")
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("NvlsFlatGrad needs an initialised process group (NCCL) for the rendezvous")
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        n_pad = (n + 3) // 4 * 4
        group = self.group if self.group is not None else dist.group.WORLD
        buf = symm_mem.empty(n_pad, dtype=torch.float32, device=dev)
        self._handle = symm_mem.rendezvous(buf, group)
        if not int(self._handle.multicast_ptr):
            raise RuntimeError("NvlsFlatGrad: no NVSwitch multicast support on this platform; use FlatGrad (NCCL)")
        buf.zero_()
        self._buf = buf
        self.flat = buf[:n]
        self.offsets, self.shapes, off = [], [], 0
        for p in self.params:
            self.offsets.append(off)
            self.shapes.append(tuple(p.shape))
            off += p.numel()
        self._bind(copy=False)
        pad_words = int(self._handle.signal_pad_size) // 4 - self.PAD_SKIP      # csrc/nvls_kernels.h NVLS_PAD_SKIP
        if pad_words < self._handle.world_size:
            raise RuntimeError("NvlsFlatGrad: signal pad too small")
        self._blocks = self.BLOCKS
        self._handle.barrier()      # everyone's buffer and pads exist (and are zero) before the first kernel

    def allreduce(self, average=True, group=None):
        import _dgm_lib
        self._bind(copy=True)
        h = self._handle
        world = h.world_size
        rc = _dgm_lib.lib().dgx_allreduce_nvls(int(h.multicast_ptr), self._buf.numel(), int(h.signal_pad_ptrs_dev),
                                               h.rank, world, self._epoch, (1.0 / world) if average else 1.0,
                                               self._blocks, _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgx_allreduce_nvls")
        self._epoch += 2
        return self.flat


def sync_densification_stats(xyz_gradient_accum, denom, max_radii2D, group=None):
    """Sum the accumulated view-space gradient norms / visit counts and take the max of the screen radii
    over ranks (two small collectives, off the per-step critical path: every densification interval)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    buf = torch.cat([xyz_gradient_accum.reshape(-1), denom.reshape(-1)])
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    n = xyz_gradient_accum.numel()
    xyz_gradient_accum.copy_(buf[:n].view_as(xyz_gradient_accum))
    denom.copy_(buf[n:].view_as(denom))
    dist.all_reduce(max_radii2D, op=dist.ReduceOp.MAX, group=group)


def broadcast_parameters(params, src=0, group=None):
    """Topology-changing steps (densify / prune / anchor) run on rank `src`; everyone else receives."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    for p in params:
        dist.broadcast(p.data, src=src, group=group)
