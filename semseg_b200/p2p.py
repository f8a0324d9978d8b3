"""SyncBatchNorm statistics exchange over NVLink peer memory (torch symmetric memory).

One process per GPU; every rank allocates the same symmetric buffer, `rendezvous` maps all peers' buffers into this
process, and the exchange kernels (csrc/bn.cu: the peer forms of bn_finalize_partials and bn_bwd_reduce_final) push
every value as one 8-byte {value, sequence number} word into every peer's buffer and poll their own memory for the peers'
words (flag-in-data, no fences, no counters) — all over NVLink — one kernel per BatchNorm exchange instead of
merge-kernel + NCCL collective + finalise-kernel.
If symmetric memory cannot be set up (no P2P access, single process, SEMSEG_B200_SYNCBN=nccl) the callers use the
NCCL path (torch.distributed all_gather / all_reduce); both paths compute the same statistics.
"""
import ctypes
import os

import torch
import torch.distributed as dist

N_SLOTS = 256                   # exchanges per epoch (PSPNet101: 224 per step); more simply open a new epoch
SLOT_FLOATS = 3 * 4096          # one rank's block: (mean, M2, n) for up to 4096 channels; a slot holds `world` of them

_exchanges = {}


class PeerExchange:
    def __init__(self, pg):
        import torch.distributed._symmetric_memory as symm_mem
        self.world = dist.get_world_size(pg)
        self.rank = dist.get_rank(pg)
        if self.world > 8:
            raise RuntimeError("peer exchange supports up to 8 ranks (one NVSwitch domain)")
        dev = torch.device("cuda", torch.cuda.current_device())
        # data words are 8 bytes ({fp32 value, sequence number}): two fp32 elements per word
        self.buf = symm_mem.empty(2 * N_SLOTS * self.world * SLOT_FLOATS, dtype=torch.float32, device=dev)
        self.buf.zero_()
        self.handle = symm_mem.rendezvous(self.buf, pg)
        self.data_ptrs = (ctypes.c_void_p * self.world)(*[int(p) for p in self.handle.buffer_ptrs])
        # Device-resident step counter = the sequence number of every exchange of the current step. The kernels read it
        # when they run, so a training step captured in a CUDA graph (slots baked in) can be replayed: the graph only
        # has to contain the increment (begin_step) once per step.
        self.step = torch.ones((1,), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        self.handle.barrier()           # every rank's buffer is zero before the first exchange
        torch.cuda.synchronize()
        self.calls = 0

    def begin_step(self, force=False):
        """Start a new exchange epoch: slots are handed out from 0 again under a new sequence number. Called at the top
        of every training forward (same point on every rank); a slot is reused only after at least one other exchange
        of the same or the following step, which orders the reuse after every peer's reads of the old contents.
        force=True (while a step is captured into a CUDA graph) issues the increment unconditionally."""
        if self.calls or force:
            self.step.add_(1)           # a (capturable) device-side increment
            self.calls = 0

    def next(self):
        """Slot of the next exchange: identical on every rank because all ranks run the same op sequence. The kernel
        takes the sequence number from the device-resident step counter."""
        if self.calls >= N_SLOTS:       # more exchanges than slots without a begin_step(): open a new epoch
            self.begin_step()
        k = self.calls
        self.calls += 1
        return k


def get_exchange(pg):
    """PeerExchange for a process group, or None when the NCCL path must be used."""
    if os.environ.get("SEMSEG_B200_SYNCBN", "p2p").lower() == "nccl":
        return None
    key = id(pg)
    if key not in _exchanges:
        ex, why = None, ""
        try:
            ex = PeerExchange(pg)
        except Exception as e:      # noqa: BLE001 - symmetric memory unsupported here: use NCCL
            why = str(e).splitlines()[0][:160] if str(e) else type(e).__name__
        # every rank must take the same path: the peer kernels and the NCCL collectives cannot be mixed
        okf = torch.tensor([1 if ex is not None else 0], dtype=torch.int32,
                           device=torch.device("cuda", torch.cuda.current_device()))
        dist.all_reduce(okf, op=dist.ReduceOp.MIN, group=pg)
        if int(okf.item()) == 0:
            if dist.get_rank(pg) == 0:
                print("semseg_b200: NVLink peer exchange unavailable on at least one rank (%s); SyncBN statistics go "
                      "through NCCL on all ranks" % (why or "a peer failed"))
            ex = None
        _exchanges[key] = ex
    return _exchanges[key]


def begin_step(pg=None, force=False):
    """Open a new exchange epoch on the (already created) peer exchange of `pg`; no-op without one."""
    if not (dist.is_available() and dist.is_initialized()):
        return
    ex = _exchanges.get(id(pg if pg is not None else dist.group.WORLD))
    if ex is not None:
        ex.begin_step(force)


def exchange_kind(pg=None):
    if not (dist.is_available() and dist.is_initialized()):
        return "none"
    pg = pg if pg is not None else dist.group.WORLD
    ex = _exchanges.get(id(pg))
    return "nvlink-p2p" if ex is not None else "nccl"
