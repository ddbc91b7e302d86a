"""Multi-GPU plumbing for the render path: one process per GPU, views sharded across ranks, ONE all-gather of
the rendered frames (SURVEY.md section 8e).  The render itself needs no collective: every frame depends on
one MPI and one pose (mpi.py:308-436 has no cross-view term).  NCCL on GPUs, gloo in the CPU tests."""
from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced [lo, hi) slice of n_items for `rank` (first n_items % world ranks get one more)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_views_mpi_major(view2mpi: List[int], rank: int, world: int) -> Tuple[int, int]:
    """Partition by MPI first, then by view (SURVEY.md 8e): whole MPIs go to one rank whenever there are at least
    as many MPIs as ranks, so d/d rgba never needs a cross-rank reduction; with fewer MPIs than ranks the views
    of an MPI are split and the (replicated) MPI's gradient must be all-reduced by the caller."""
    n_mpi = (max(view2mpi) + 1) if len(view2mpi) else 0
    if n_mpi >= world:
        m_lo, m_hi = shard_range(n_mpi, rank, world)
        idx = [i for i, m in enumerate(view2mpi) if m_lo <= m < m_hi]
        return (idx[0], idx[-1] + 1) if idx else (0, 0)
    return shard_range(len(view2mpi), rank, world)


def pack_frames(color: torch.Tensor, depth: torch.Tensor) -> torch.Tensor:
    """[V,3,H,W] + [V,1,H,W] -> [V,4,H,W] (RGB + depth = one 'frame', 16*H*W bytes)."""
    return torch.cat([color, depth], dim=1)


def all_gather_frames(frames: torch.Tensor, counts: List[int] = None, group=None) -> torch.Tensor:
    """Gather every rank's [V_r,4,H,W] frames into [sum V_r,4,H,W] on every rank, rank-major (= view order when
    views were sharded with shard_range).  Equal counts use one all_gather_into_tensor (ncclAllGather);
    ragged counts pad to the max and slice."""
    world = dist.get_world_size(group)
    if world == 1:
        return frames
    if counts is None:
        counts = [frames.shape[0]] * world
    vmax = max(counts)
    if all(c == vmax for c in counts):
        out = torch.empty((world * vmax,) + tuple(frames.shape[1:]), dtype=frames.dtype, device=frames.device)
        dist.all_gather_into_tensor(out, frames.contiguous(), group=group)
        return out
    pad = torch.zeros((vmax,) + tuple(frames.shape[1:]), dtype=frames.dtype, device=frames.device)
    pad[: frames.shape[0]] = frames
    out = torch.empty((world * vmax,) + tuple(frames.shape[1:]), dtype=frames.dtype, device=frames.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return torch.cat([out[r * vmax: r * vmax + counts[r]] for r in range(world)], dim=0)


class FrameGather:
    """All-gather of rendered frames fused into the render kernel (SURVEY.md 8e, the one collective of the path).

    Every rank owns symmetric-memory buffers [world * frames_per_rank, 4, H, W] that all peers map over NVLink
    (torch.distributed._symmetric_memory).  `render()` launches the forward kernel with the peers' buffer pointers: the
    epilogue stores each finished pixel into frame slot rank * frames_per_rank + v of EVERY rank's buffer, so the gather
    overlaps the render tile by tile (posted NVLink writes) instead of following it as a separate ncclAllGather;
    `finish()` is the device-side barrier that makes the remote stores visible.  `frames` is then the gathered tensor.

    Ordering (write-after-read across iterations).  The buffers are DOUBLE-BUFFERED: step k writes buffer k % 2.  A peer
    may start step k+2 (which overwrites buffer k % 2 on every rank) only after it passed barrier k+1, and barrier k+1
    completes on a rank only when that rank's stream has reached its own `finish()` of step k+1.  So every kernel that reads
    `frames` of step k is safe provided it was enqueued ON THE RENDER STREAM (or on a stream the render stream waits on)
    before the next `finish()` -- the natural program order render, finish, consume, render, finish, ...  A consumer on an
    unrelated stream must be joined to the render stream first.  (Round 1 had one buffer and only the trailing barrier: a fast
    rank's step k+1 could overwrite frames a slow rank was still reading; tests/test_gpu_multi.py renders different data
    per step with a reader in flight to cover this.)
    """

    def __init__(self, frames_per_rank: int, H: int, W: int, device, group=None, multicast="auto"):
        """multicast: "auto" (use the NVLS multicast mapping of the buffers when the fabric offers one), True (require it), False
        (per-peer stores).  With a multicast address the epilogue issues ONE float4 store per quad and the NVSwitch replicates it
        to every rank's buffer; without, n_peers stores."""
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.frames_per_rank, self.H, self.W = frames_per_rank, H, W
        self._bufs, self._handles, self._peer_ptrs = [], [], []
        self.multicast = False
        for _ in range(2):
            buf = symm_mem.empty((self.world * frames_per_rank, 4, H, W), dtype=torch.float32, device=device)
            handle = symm_mem.rendezvous(buf, self.group)
            ptrs = [int(p) for p in handle.buffer_ptrs]
            assert len(ptrs) == self.world
            mc = int(getattr(handle, "multicast_ptr", 0) or 0)
            if multicast is True and mc == 0:
                raise RuntimeError("FrameGather(multicast=True): the symmetric-memory handle has no multicast mapping (no NVLS)")
            if multicast and mc != 0:
                ptrs, self.multicast = [mc], True
            self._bufs.append(buf)
            self._handles.append(handle)
            self._peer_ptrs.append(torch.tensor(ptrs, dtype=torch.int64, device=device))   # device array of float* (peers, or the multicast address)
        self._next, self._done = 0, None

    @property
    def frames(self) -> torch.Tensor:
        """The gathered frames of the most recently finished step ([world * frames_per_rank, 4, H, W])."""
        assert self._done is not None, "no finished step yet: call render() and finish() first"
        return self._bufs[self._done]

    def render(self, rgba, dhw, view2mpi, ray_dir, eye, z_dir, flags, *, align_corners=True, check_last_plane=False,
               color_minus1_1=False, early_stop=None):
        """early_stop: early ray termination threshold in [0, 1), as in render_frames (None: off).  An fp16 rgba renders natively
        where render_frames would (GMPI_MPI_F16), else from its fp32 upcast."""
        from . import _lib
        from .mpi import _launch_mpi, _mpi_desc, _options, _render_fwd
        _lib.load()                     # a missing library is reported before the arguments are checked
        V = ray_dir.shape[0]
        assert rgba.ndim == 5 and V <= self.frames_per_rank and ray_dir.shape[2:] == (self.H, self.W)
        options = _options(align_corners, check_last_plane, color_minus1_1, early_stop=early_stop)
        if rgba.dtype == torch.float16:     # any other MPI is rendered as passed (asserted below)
            (rgba, _, _, _), options = _launch_mpi([rgba, None, None, None], V, self.H, self.W, options)
        mpi_dtype = torch.float16 if options & _lib.OPT_MPI_F16 else torch.float32
        f32 = torch.float32
        for name, t, dtype in (("rgba", rgba, mpi_dtype), ("dhw", dhw, f32), ("ray_dir", ray_dir, f32), ("eye", eye, f32),
                               ("z_dir", z_dir, f32)):   # raw pointers below
            assert t.is_cuda and t.dtype == dtype and t.is_contiguous(), f"{name} must be a contiguous {dtype} CUDA tensor"
        assert view2mpi.dtype == torch.int32 and view2mpi.is_contiguous() and flags.dtype == torch.int32
        peers = self._peer_ptrs[self._next]
        _render_fwd(_mpi_desc([rgba, None, None, None], V, self.H, self.W, options, view2mpi=view2mpi, dhw=dhw, ray_dir=ray_dir,
                              eye=eye, z_dir=z_dir, peer_frames=peers, n_peers=int(peers.numel()),
                              frame_offset=self.rank * self.frames_per_rank, flags=flags, early_stop=early_stop), None, rgba.device)

    def finish(self):
        """Barrier across ranks on the current stream: after it, every rank's `frames` holds all ranks' frames."""
        self._handles[self._next].barrier(channel=0)
        self._done = self._next
        self._next ^= 1
