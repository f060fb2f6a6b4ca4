"""Multi-GPU plumbing: utterances are independent, so the path shards by utterance
with NO collective on the hot path (SURVEY.md §8e).  The only communication is
one broadcast of the packed weight blobs from rank 0 at start-up
(torch.distributed, NCCL over NVLink on GPUs / gloo in the CPU tests)."""
from __future__ import annotations

import numpy as np


def lpt_shard(costs, world_size: int):
    """Longest-processing-time-first assignment of utterances to ranks.
    costs: per-utterance cost (n_frames).  Returns list (len world_size) of index lists,
    each sorted by decreasing cost so that length buckets stay contiguous."""
    costs = np.asarray(costs, dtype=np.int64)
    order = np.argsort(-costs, kind="stable")
    loads = np.zeros(world_size, dtype=np.int64)
    shards = [[] for _ in range(world_size)]
    for i in order:
        r = int(np.argmin(loads))
        shards[r].append(int(i))
        loads[r] += int(costs[i])
    return shards


def bucket_by_length(n_frames, max_pad_frac: float = 0.08, max_rows: int = 128):
    """Group utterance indices (any order) into batches whose padding overhead
    (rows padded to the longest member) stays below max_pad_frac.  Returns list of index lists."""
    n_frames = np.asarray(n_frames, dtype=np.int64)
    order = list(np.argsort(-n_frames, kind="stable"))
    buckets, cur = [], []
    for i in order:
        if not cur:
            cur = [int(i)]
            continue
        longest = int(n_frames[cur[0]])
        total = int(n_frames[cur].sum() + n_frames[i])
        padded = longest * (len(cur) + 1)
        if len(cur) < max_rows and (padded - total) <= max_pad_frac * padded:
            cur.append(int(i))
        else:
            buckets.append(cur)
            cur = [int(i)]
    if cur:
        buckets.append(cur)
    return buckets


# cost model of one ragged batch, used only to balance buckets (relative weights): the decoder scan is paid per frame of
# the batch's longest row (sequential, ~20 us per frame for up to 32 rows), everything else per padded row-frame
SCAN_US_PER_FRAME = 17.0          # + SCAN_US_PER_FRAME_ROW per row of the launch
SCAN_US_PER_FRAME_ROW = 0.15
ROW_US_PER_FRAME = 1.9


def batch_cost_us(n_frames_of_rows) -> float:
    n = np.asarray(n_frames_of_rows, dtype=np.int64)
    rows = len(n)
    scans = (rows + 31) // 32                         # row groups of 32 (one launch takes up to 4; they share its barriers, so this
                                                      # over-estimates > 32 rows by ~10 %: balanced_buckets keeps buckets <= 32 rows)
    return float(n.max()) * (SCAN_US_PER_FRAME * scans + SCAN_US_PER_FRAME_ROW * rows + ROW_US_PER_FRAME * rows)


def balanced_buckets(n_frames, world_size: int, groups_per_rank=None, max_pad_frac: float = 0.08, max_rows: int = 32):
    """Mixed-length workload (BASELINE configs[4]) for `world_size` ranks: utterances sorted by frame count are cut into
    world_size * groups_per_rank CONTIGUOUS buckets of (nearly) equal predicted cost -- so a bucket of long utterances
    has fewer rows than one of short ones -- and the buckets are LPT-assigned to the ranks.  With equal-cost buckets and
    a bucket count that is a multiple of the rank count the assignment is balanced by construction, which plain
    `bucket_by_length` + `lpt_shard` is not when there are only ~2 buckets per rank.  `max_pad_frac` bounds the padding
    of the WHOLE workload (padded row-frames vs real frames); if the equal-cost cut exceeds it, more buckets per rank are
    used.  groups_per_rank=None tries 2, 3 and 4 and keeps the cut with the smallest predicted makespan.
    Returns (buckets: list of index lists, shards: list (len world_size) of bucket-index lists)."""
    if groups_per_rank is None:
        best = None
        for g_ in (2, 3, 4):
            b_, s_ = balanced_buckets(n_frames, world_size, g_, max_pad_frac, max_rows)
            nn = np.asarray(n_frames, dtype=np.int64)
            span = max(sum(batch_cost_us(nn[b_[i]]) for i in sh) for sh in s_)
            if best is None or span < best[0]:
                best = (span, b_, s_)
        return best[1], best[2]
    n = np.asarray(n_frames, dtype=np.int64)
    order = [int(i) for i in np.argsort(-n, kind="stable")]

    def pack(cap_us):
        """Greedy contiguous packing under a per-bucket cost cap (and the row limit of one decoder scan)."""
        out, cur = [], []
        for i in order:
            cand = cur + [i]
            if cur and (len(cand) > max_rows or batch_cost_us(n[cand]) > cap_us):
                out.append(cur)
                cur = [i]
            else:
                cur = cand
        if cur:
            out.append(cur)
        return out

    g = groups_per_rank
    while True:
        G = max(1, world_size * g)
        # smallest cost cap that needs at most G buckets: every bucket then costs about the same (<= cap)
        lo, hi = float(batch_cost_us(n[order[:1]])), float(batch_cost_us(n[order])) + 1.0
        for _ in range(40):
            mid = 0.5 * (lo + hi)
            if len(pack(mid)) <= G:
                hi = mid
            else:
                lo = mid
        buckets = pack(hi)
        padded = sum(len(b) * int(n[b[0]]) for b in buckets)
        if 1.0 - float(n.sum()) / padded <= max_pad_frac or G >= len(order):
            break
        g += 1
    shards = lpt_shard([int(batch_cost_us(n[b])) for b in buckets], world_size)
    return buckets, shards


def broadcast_blob(blob_np, device, src: int = 0, group=None):
    """Broadcast a float32 blob from rank `src`; returns a torch tensor on `device`
    on every rank.  `blob_np` is only read on rank `src` (other ranks pass the size)."""
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if rank == src:
        t = torch.from_numpy(np.ascontiguousarray(blob_np, dtype=np.float32)).to(device)
    else:
        n = int(blob_np) if np.isscalar(blob_np) else int(np.asarray(blob_np).size)
        t = torch.empty(n, dtype=torch.float32, device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(t, src=src, group=group)
    return t


def load_weights_distributed(engine, hifigan_params=None, acoustic_ckpt=None, device=None, src: int = 0, group=None,
                             duration_ckpt=None, with_duration: bool = False):
    """Rank `src` packs the Haiku-layout checkpoints; every rank receives the packed
    blobs by one broadcast each and loads them from DEVICE memory (no host round trip).
    `with_duration` (same value on every rank) adds the duration model's blob (SURVEY.md §8e: 55.7 + 50.1 + 7.4 MB)."""
    import torch
    import torch.distributed as dist

    from . import _lib, weights

    rank = dist.get_rank(group) if dist.is_initialized() else 0
    lib = _lib.load()
    device = device if device is not None else torch.device("cuda", engine.device)
    hb = weights.pack_hifigan(hifigan_params) if rank == src else int(lib.vtts_hifigan_blob_floats())
    ab = weights.pack_acoustic(acoustic_ckpt) if rank == src else int(lib.vtts_acoustic_blob_floats())
    ht = broadcast_blob(hb, device, src, group)
    at = broadcast_blob(ab, device, src, group)
    torch.cuda.synchronize(device)
    engine.load_hifigan(ht)
    engine.load_acoustic(at)
    total = ht.numel() * 4 + at.numel() * 4
    if with_duration or duration_ckpt is not None:
        db = weights.pack_duration(duration_ckpt) if rank == src else int(lib.vtts_duration_blob_floats())
        dt = broadcast_blob(db, device, src, group)
        torch.cuda.synchronize(device)
        engine.load_duration(dt)
        total += dt.numel() * 4
    return total


# ---------------------------------------------------------------------------------------------------------
# start-up broadcast through the C ABI (vtts_broadcast_weights): for hosts that are not Python / torch the ABI call
# is the whole story (they hand in their own ncclComm_t); this helper builds a communicator for the torch case.
# ---------------------------------------------------------------------------------------------------------
class NcclComm:
    """A raw ncclComm_t over the ranks of the initialised torch.distributed group, created with ctypes on the libnccl
    the process already has loaded (torch's bundled copy).  The unique id travels through torch.distributed."""

    def __init__(self, device_index: int, group=None):
        import ctypes as C
        import torch
        import torch.distributed as dist

        path = None
        with open("/proc/self/maps") as f:
            for line in f:
                if "libnccl.so" in line:
                    path = line.split()[-1]
                    break
        self.lib = C.CDLL(path or "libnccl.so.2")

        class UniqueId(C.Structure):
            _fields_ = [("internal", C.c_char * 128)]

        self.lib.ncclGetUniqueId.argtypes = [C.POINTER(UniqueId)]
        self.lib.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, UniqueId, C.c_int]
        self.lib.ncclCommDestroy.argtypes = [C.c_void_p]
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        uid = UniqueId()
        if rank == 0:
            rc = self.lib.ncclGetUniqueId(C.byref(uid))
            if rc != 0:
                raise RuntimeError(f"ncclGetUniqueId -> {rc}")
        box = [bytes(uid.internal)] if rank == 0 else [None]
        # bytes() of a c_char array stops at the first NUL: ship the raw buffer instead
        box = [C.string_at(C.addressof(uid), 128)] if rank == 0 else [None]
        dist.broadcast_object_list(box, src=0, group=group)
        C.memmove(C.addressof(uid), box[0], 128)
        torch.cuda.set_device(device_index)
        comm = C.c_void_p()
        rc = self.lib.ncclCommInitRank(C.byref(comm), world, uid, rank)
        if rc != 0:
            raise RuntimeError(f"ncclCommInitRank -> {rc}")
        self.handle = comm
        self.rank, self.world = rank, world

    def close(self):
        if getattr(self, "handle", None):
            self.lib.ncclCommDestroy(self.handle)
            self.handle = None


def load_weights_via_abi(engine, hifigan_params=None, acoustic_ckpt=None, duration_ckpt=None, src: int = 0, group=None):
    """Rank `src` loads the Haiku-layout checkpoints into its context; every other rank receives them by
    vtts_broadcast_weights (one grouped ncclBroadcast of the device arenas).  Returns the NcclComm (keep or close)."""
    import torch.distributed as dist
    rank = dist.get_rank(group)
    if rank == src:
        if hifigan_params is not None:
            engine.load_hifigan(hifigan_params)
        if acoustic_ckpt is not None:
            engine.load_acoustic(acoustic_ckpt)
        if duration_ckpt is not None:
            engine.load_duration(duration_ckpt)
    comm = NcclComm(engine.device, group)
    engine.broadcast_weights(comm.handle, src, rank == src)
    return comm
