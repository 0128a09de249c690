"""Multi-GPU plumbing (SURVEY section 8e): envs are independent, so the env index range is split
into contiguous shards, one process per GPU, and the only collective on the step path is one
all-gather of the observation tensor for the policy.  The reference has no distributed code;
there is nothing to be compatible with.  Backend-agnostic (nccl on GPUs, gloo in CPU tests)."""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(num_envs_global: int, rank: int, world_size: int) -> Tuple[int, int]:
    """(offset, count) of the contiguous shard of ``rank``; the remainder goes to the first ranks."""
    if not (0 <= rank < world_size):
        raise ValueError("rank out of range")
    base, rem = divmod(num_envs_global, world_size)
    count = base + (1 if rank < rem else 0)
    offset = rank * base + min(rank, rem)
    return offset, count


def env_from_torchrun():
    """(rank, local_rank, world_size) from the torchrun environment (defaults: single process)."""
    return int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


class ObsAllGather:
    """Persistent buffers for the per-step observation all-gather.

    Equal shards use ``all_gather_into_tensor`` (one NCCL kernel into a contiguous [N,D] buffer);
    ragged shards (N not divisible by the world size) gather max-count padded blocks and compact."""

    def __init__(self, local_count: int, feat: int, num_envs_global: int, device, dtype=torch.float32,
                 group: Optional[dist.ProcessGroup] = None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.out = torch.empty(num_envs_global, feat, device=device, dtype=dtype)
        counts = [shard_range(num_envs_global, r, self.world)[1] for r in range(self.world)]
        if counts[self.rank] != local_count:
            raise ValueError(f"rank {self.rank}: local shard has {local_count} envs, expected {counts[self.rank]}")
        self.equal = len(set(counts)) == 1
        self.offs = [shard_range(num_envs_global, r, self.world)[0] for r in range(self.world)]
        self.counts = counts
        if not self.equal:
            self.pad_in = torch.zeros(max(counts), feat, device=device, dtype=dtype)
            self.pad_out = torch.empty(self.world * max(counts), feat, device=device, dtype=dtype)

    def __call__(self, obs_local: torch.Tensor) -> torch.Tensor:
        if self.world == 1:
            self.out.copy_(obs_local)
        elif self.equal:
            dist.all_gather_into_tensor(self.out, obs_local.contiguous(), group=self.group)
        else:
            mc = self.pad_in.shape[0]
            self.pad_in[: obs_local.shape[0]].copy_(obs_local)
            dist.all_gather_into_tensor(self.pad_out, self.pad_in, group=self.group)
            for r, (o, c) in enumerate(zip(self.offs, self.counts)):
                self.out[o:o + c].copy_(self.pad_out[r * mc: r * mc + c])
        return self.out


class P2PObsAllGather:
    """Same contract as ObsAllGather (equal shards only), but the collective is ONE hand-written
    kernel of NVLink peer stores + a flag handshake (csrc/p2p_allgather.cu) over buffers obtained
    from a torch symmetric-memory rendezvous -- no NCCL call on the step path."""

    def __init__(self, local_count: int, feat: int, device, group=None, dtype=torch.float32, num_buffers: int = 2):
        import ctypes as C

        import torch.distributed._symmetric_memory as symm_mem

        from . import _lib

        self._C, self._lib = C, _lib.load()
        self._check = _lib.check
        group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if dtype != torch.float32:
            raise ValueError("float32 only")
        self.bytes = local_count * feat * 4
        if self.bytes % 16:
            raise ValueError("shard bytes must be a multiple of 16")
        self.device = torch.device(device)
        # two gathered buffers, alternated by epoch parity: a peer can run at most one epoch ahead of
        # the slowest reader (everybody waits for everybody's flag), so epoch e+1 never overwrites
        # data of epoch e that a slower rank may still be consuming
        # (fused mode with lag 1 needs 4: a rank may push epoch e+4 once its peers finished epoch e+2,
        # i.e. after their consumers of epoch e -- stream-ordered before their step e+2 -- are done)
        if num_buffers not in (2, 4):
            raise ValueError("num_buffers must be 2 or 4")
        self.num_buffers = num_buffers
        self.outs, self.buf_ptrs = [], []
        for _ in range(num_buffers):
            o = symm_mem.empty(self.world * local_count, feat, dtype=dtype, device=self.device)
            h = symm_mem.rendezvous(o, group)
            self.outs.append(o)
            self.buf_ptrs.append(torch.tensor(list(h.buffer_ptrs), dtype=torch.int64, device=self.device))
            setattr(self, f"_h{len(self.outs)}", h)
        self.flags = symm_mem.empty(64, dtype=torch.int32, device=self.device)
        self.flags.zero_()
        self.h_flags = symm_mem.rendezvous(self.flags, group)
        self.flag_ptrs = torch.tensor(list(self.h_flags.buffer_ptrs), dtype=torch.int64, device=self.device)
        self.scratch = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.epoch = 0
        torch.cuda.synchronize(self.device)
        dist.barrier(group)  # every rank's flags are zeroed before anybody publishes epoch 1

    def next_epoch(self):
        """(epoch, buffer parity) of the next collective -- used by Hp1Engine when the all-gather is
        fused into the step kernel (Hp1Engine.attach_obs_gather)."""
        self.epoch += 1
        return self.epoch, self.epoch % self.num_buffers

    def __call__(self, obs_local: torch.Tensor) -> torch.Tensor:
        C = self._C
        if obs_local.numel() * 4 != self.bytes or not obs_local.is_contiguous():
            raise ValueError("obs_local must be the contiguous local shard")
        _, b = self.next_epoch()
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        self._check(self._lib.agx_p2p_allgather(
            C.c_void_p(obs_local.data_ptr()), C.c_void_p(self.buf_ptrs[b].data_ptr()), C.c_void_p(self.flag_ptrs.data_ptr()),
            self.world, self.rank, C.c_uint64(self.bytes), C.c_uint32(self.epoch), C.c_void_p(self.scratch.data_ptr()), stream),
            "agx_p2p_allgather")
        return self.outs[b]


class PipelinedObsGather:
    """The observation all-gather of SURVEY 8e as two hand-written kernels that run BESIDE the steps instead of inside them
    (csrc/p2p_allgather.cu: agx_obs_gather_push / agx_obs_gather_wait), over a ring of `num_buffers` symmetric-memory buffers:

    * sender: the step writes its observation straight into this rank's slot of ring buffer `epoch % num_buffers`; `push`
      (that ring slot's own side stream, <= max_ctas CTAs that fit beside the resident step kernel) stores it into the same place
      of every peer's buffer over NVLink and, once its stores have been performed, publishes `epoch` in every rank's flag word of
      that ring slot.  Pushes into different ring slots run concurrently: one push alone is a chain of latencies (wake-up, L2
      reads, NVLink drain, two system fences: ~15 us for 3.4 MB), `num_buffers` of them in flight sustain a step period of a
      few microseconds;
    * receiver: `wait(epoch)` = a one-warp kernel on the consumer's stream that retires when all `world` flags show `epoch`.

    The push never waits for a peer and the step kernel never waits for anything of this class.  Re-use of a ring slot is ordered by a
    one-warp GATE kernel that `next_epoch()` puts in front of the step (agx_obs_gather_gate, programmatic stream serialization): it
    lets the step launch in only when the push that last read the slot has finished reading -- the chained step launches stay
    chained (no event, no stream-level wait), and a step that has to wait is not resident while it waits.  Equal shards only.
    Consumer side: nothing holds a PEER back, so the gathered buffer of epoch e may be overwritten by a peer's push of epoch
    e + num_buffers.  A consumer that waits every step (the task API: the policy needs the observation) keeps the ranks within one
    step of each other -- a rank's step e + 1 needs its own wait(e), i.e. every peer's push e -- so num_buffers >= 2 suffices; a
    free-running producer (bench.py's timed loop) may only read the epoch it finally waits for.
    `loopback_world` (tests, one GPU): emulate a world of that size inside one process -- every "peer" buffer is a local
    buffer, rank 0 is this process; the protocol (ring, flags, counters) runs exactly as on several GPUs."""

    def __init__(self, local_count: int, feat: int, device, group=None, num_buffers: int = 4, max_ctas: int = 24,
                 loopback_world: int = 0, multicast: Optional[bool] = None):
        """multicast: push through the NVSwitch multicast address of the ring buffers (`multimem.st`: every 16 bytes leave the GPU once,
        the switch replicates) when the symmetric-memory rendezvous offers one; None = the AGX_GATHER_MULTICAST environment variable if
        set, else on for a world of 3 or more ranks"""
        import ctypes as C

        from . import _lib

        self._C, self._lib, self._check = C, _lib.load(), _lib.check
        self.device = torch.device(device)
        if not 1 <= int(num_buffers) <= 4:
            raise ValueError("num_buffers must be in [1, 4] (flag words: 4 ring slots x AGX_MAX_PEERS)")
        self.num_buffers, self.max_ctas = int(num_buffers), int(max_ctas)
        self.bytes = local_count * feat * 4
        if self.bytes % 16:
            raise ValueError("shard bytes must be a multiple of 16")
        self.local_count, self.feat = local_count, feat
        i64 = lambda ptrs: torch.tensor(list(ptrs), dtype=torch.int64, device=self.device)
        self._handles, self.mc_ptrs = [], []
        if multicast is None:
            env = os.environ.get("AGX_GATHER_MULTICAST")
            multicast = (env != "0") if env is not None else None
        B = self.num_buffers
        if loopback_world:
            self.world, self.rank = int(loopback_world), 0
            self.outs = [torch.zeros(self.world * local_count, feat, device=self.device) for _ in range(B)]
            # "peer" p's gathered buffers: separate local tensors (peer 0 = ours)
            self.peer_outs = [[self.outs[b]] + [torch.zeros_like(self.outs[b]) for _ in range(self.world - 1)] for b in range(B)]
            self.buf_ptrs = [i64(t.data_ptr() for t in self.peer_outs[b]) for b in range(B)]
            self.flags = torch.zeros(64, dtype=torch.int32, device=self.device)
            self.peer_flags = [self.flags] + [torch.zeros_like(self.flags) for _ in range(self.world - 1)]
            self.flag_ptrs = i64(t.data_ptr() for t in self.peer_flags)
        else:
            import torch.distributed._symmetric_memory as symm_mem

            group = group if group is not None else dist.group.WORLD
            self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
            self.outs, self.buf_ptrs = [], []
            for _ in range(B):
                o = symm_mem.empty(self.world * local_count, feat, dtype=torch.float32, device=self.device)
                h = symm_mem.rendezvous(o, group)
                o.zero_()
                self.outs.append(o)
                self.buf_ptrs.append(i64(h.buffer_ptrs))
                self._handles.append(h)
                self.mc_ptrs.append(int(getattr(h, "multicast_ptr", 0) or 0))
            self.flags = symm_mem.empty(64, dtype=torch.int32, device=self.device)
            self.flags.zero_()
            h = symm_mem.rendezvous(self.flags, group)
            self._handles.append(h)
            self.flag_ptrs = i64(h.buffer_ptrs)
        r0 = self.rank * local_count
        self.own_slot = [o[r0:r0 + local_count] for o in self.outs]
        self.own_slot_ptr = [t.data_ptr() for t in self.own_slot]
        self.scratch = torch.zeros(B, 4, dtype=torch.int32, device=self.device)
        self.error_word = torch.zeros(1, dtype=torch.int32, device=self.device)
        # one side stream + one event per ring slot; high priority: their few CTAs go ahead of the next step's
        self.streams = [torch.cuda.Stream(device=self.device, priority=-1) for _ in range(B)]
        self._raw = [st.cuda_stream for st in self.streams]
        self.events = [torch.cuda.Event() for _ in range(B)]
        self._pending = [False] * B
        self.read_done = torch.zeros(B, dtype=torch.int32, device=self.device)  # per ring slot: epoch of the last push that finished reading
        self._pushes = []
        for b in range(B):
            a = _lib.AgxObsGatherPush()
            a.peer_bufs, a.peer_flags, a.world, a.rank = self.buf_ptrs[b].data_ptr(), self.flag_ptrs.data_ptr(), self.world, self.rank
            a.bytes, a.max_ctas, a.flag_slot = self.bytes, self.max_ctas, b
            a.scratch, a.error_word = self.scratch[b].data_ptr(), self.error_word.data_ptr()
            a.read_done = self.read_done[b].data_ptr()
            use_mc = (self.world >= 3) if multicast is None else bool(multicast)
            a.mc_buf = (self.mc_ptrs[b] or None) if (use_mc and len(self.mc_ptrs) == B and all(self.mc_ptrs)) else None
            self._pushes.append((a, C.byref(a)))
        self.multicast = bool(self._pushes[0][0].mc_buf)
        self.epoch = 0
        self._read_done_ptr = [self.read_done[b].data_ptr() for b in range(B)]
        self._err_ptr = self.error_word.data_ptr()
        torch.cuda.synchronize(self.device)
        if not loopback_world:
            dist.barrier(group)  # every rank's flags are zeroed before anybody publishes epoch 1

    def next_epoch(self):
        """(epoch, ring slot) of the next step.  The step will overwrite this rank's rows in ring buffer `slot`: a gate kernel in
        front of it (current stream) holds it back until the push that last read them has finished reading."""
        self.epoch += 1
        slot = self.epoch % self.num_buffers
        if self.epoch > self.num_buffers:
            rc = self._lib.agx_obs_gather_gate(self._read_done_ptr[slot], self.epoch - self.num_buffers, self._err_ptr,
                                               torch.cuda.current_stream(self.device).cuda_stream)
            if rc:
                self._check(rc, "agx_obs_gather_gate")
        return self.epoch, slot

    def push(self, local_ptr: int, epoch: int, slot: int, ready_ctr: int = 0, ready_target: int = 0, stream=None):
        """enqueue the push of `local_ptr` (this rank's rows, device pointer) as `epoch` into ring slot `slot`: on the slot's side
        stream (the kernel spins on *ready_ctr >= ready_target before reading) or, with `stream`, in that stream's order"""
        a, ref = self._pushes[slot]
        a.local, a.epoch = local_ptr, epoch
        a.ready_ctr, a.ready_target = (ready_ctr or None), ready_target
        rc = self._lib.agx_obs_gather_push(ref, self._raw[slot] if stream is None else stream)
        if rc:
            self._check(rc, "agx_obs_gather_push")
        if stream is None:
            self._pending[slot] = True

    def wait(self, epoch: Optional[int] = None, stream=None):
        """make `stream` (default: the current one) wait until every rank's rows of `epoch` (default: the latest) are here;
        returns the gathered [world*N, feat] buffer of that epoch"""
        epoch = self.epoch if epoch is None else epoch
        st = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        slot = epoch % self.num_buffers
        self._check(self._lib.agx_obs_gather_wait(self.flags.data_ptr(), slot, self.world, epoch, self.error_word.data_ptr(), st),
                    "agx_obs_gather_wait")
        return self.outs[slot]

    def fence(self):
        """the current stream waits for every push enqueued so far (before anything overwrites what a push may still read)"""
        cur = torch.cuda.current_stream(self.device)
        for b in range(self.num_buffers):
            if self._pending[b]:
                self.events[b].record(self.streams[b])
                cur.wait_event(self.events[b])
                self._pending[b] = False

    def check(self):
        """synchronise and raise if a push / wait gave up (AGX_E_TIMEOUT)"""
        self.fence()
        self._check(self._lib.agx_obs_gather_check(self.error_word.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream),
                    "agx_obs_gather_check")

    def loopback_complete(self, epoch: int):
        """loopback only: play the other ranks -- their rows are not simulated, only their flags of this epoch's ring slot"""
        slot = epoch % self.num_buffers
        for q in range(1, self.world):
            self.flags[slot * 16 + q] = epoch
