"""Host-side logic of the disparity-sharded (multi-GPU) path: which global disparity slices a rank
owns, the one exchange step of the path (per-pixel packed minima -> final maps) and the banded image
upload that keeps the per-rank PCIe traffic constant as ranks are added.

One process per GPU; `torch.distributed` supplies rendezvous and the library collectives (NCCL on
GPUs, gloo in the CPU tests).  Device work stays in the C-ABI (include/prime_stereo_b200.h).
Reference counterpart: the reference shards nothing (single process); its unit of parallel work is the
disparity slice (src/DispEst.cpp:235-268), which is what is sharded here (SURVEY.md section 8e).
"""
import ctypes as C

from . import capi


def shard_range(max_disp, world, rank, min_disp=0):
    """Contiguous slices [d_begin, d_begin + d_count) of rank `rank` in [min_disp, max_disp); the last rank takes the
    remainder.  Every rank owns at least one slice (world <= max_disp - min_disp)."""
    n = max_disp - min_disp
    if not (0 <= rank < world) or not (0 <= min_disp < max_disp) or world > n:
        raise ValueError(f"bad shard request rank={rank} world={world} range=[{min_disp},{max_disp})")
    base = n // world
    d_begin = min_disp + rank * base
    d_count = base if rank < world - 1 else max_disp - d_begin
    return d_begin, d_count


def band_rows(height, world, rank):
    """Row band [r0, r1) of the images that rank `rank` uploads; bands are equal-sized (the last may be short)."""
    rows = (height + world - 1) // world
    return min(height, rank * rows), min(height, (rank + 1) * rows), rows


def bind_to_current_stream(de):
    """Run every launch of `de` on torch's CURRENT stream, so that collectives torch issues (which are ordered
    on that stream) are ordered against the context's kernels.  The legacy default stream (handle 0) is passed
    as cudaStreamLegacy (0x1) because a NULL handle means 'the context's own stream' to psm_set_stream."""
    import torch
    h = torch.cuda.current_stream().cuda_stream
    capi.check(capi.lib().psm_set_stream(de.handle, C.c_void_p(h if h else 1)), de.handle)


def _wide(de):
    """the context has 16-bit maps (DispEst(..., map_bits=16) or maxDis > 256)"""
    return getattr(de, "map_bits", 8) == 16


def gather_and_reduce(de, keys, gathered, world, lmap=None, rmap=None, group=None):
    """Library baseline of the exchange.  keys: int64 CUDA tensor [2, H*W] (this rank's packed minima, written by
    psm_disp_select_keys); gathered: int64 CUDA tensor [2, world, H*W].  One all-gather per view, then the final
    min -> maps (u8, or u16 when de.map_bits == 16; optionally copied to host arrays).  The context is bound to torch's current stream first:
    the all-gathers must not overtake the select kernels."""
    import torch.distributed as dist
    L = capi.lib()
    bind_to_current_stream(de)
    capi.check(L.psm_disp_select_keys(de.handle, keys[0].data_ptr(), keys[1].data_ptr()), de.handle)
    dist.all_gather_into_tensor(gathered[0].view(-1), keys[0], group=group)
    dist.all_gather_into_tensor(gathered[1].view(-1), keys[1], group=group)
    lp = lmap.ctypes.data_as(C.c_void_p) if lmap is not None else None
    rp = rmap.ctypes.data_as(C.c_void_p) if rmap is not None else None
    reduce = L.psm_disp_reduce_keys_u16 if _wide(de) else L.psm_disp_reduce_keys
    step = de.wid * (2 if _wide(de) else 1)
    capi.check(reduce(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), world, lp, step, rp, step), de.handle)


class P2PExchange:
    """Sharded WTA fused with its exchange over NVLink peer memory (see include/prime_stereo_b200.h):
    select() = WTA + scatter of packed minima into the reducers' blocks, reduce() = chunk min + gather of the u8
    result into every rank's map, fetch() = D2H.  The kernels order themselves across ranks with device-side
    ARRIVE / DONE flags in the exchange blocks: a frame needs no collective and no host barrier.
    Exchange blocks are shared between the per-GPU processes through CUDA IPC handles exchanged once.
    device_sync=False falls back to caller-side barriers (a 1-element all-reduce on the context's stream)."""

    def __init__(self, de, world, rank, group=None, device_sync=True):
        import torch
        import torch.distributed as dist
        self.de, self.world, self.rank, self.group = de, world, rank, group
        self.device_sync = bool(device_sync)
        L = capi.lib()
        bind_to_current_stream(de)   # the setup collectives below and (without device_sync) the barriers share its stream
        capi.check(L.psm_set_option(de.handle, capi.PSM_OPT_P2P_SYNC, int(self.device_sync)), de.handle)
        own = C.c_void_p()
        capi.check(L.psm_p2p_create_buffer(de.handle, world, C.byref(own)), de.handle)
        handle = C.create_string_buffer(64)
        capi.check(L.psm_ipc_export(de.handle, own, handle), de.handle)
        mine = torch.frombuffer(bytearray(handle.raw), dtype=torch.uint8).cuda()
        allh = torch.empty((world, 64), dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(allh.view(-1), mine, group=group)
        allh = allh.cpu().numpy()
        ptrs = (C.c_void_p * world)()
        for r in range(world):
            if r == rank:
                ptrs[r] = own.value
            else:
                p = C.c_void_p()
                capi.check(L.psm_ipc_import(de.handle, allh[r].tobytes(), C.byref(p)), de.handle)
                ptrs[r] = p.value
        capi.check(L.psm_p2p_set_peers(de.handle, ptrs, world, rank), de.handle)
        self._flag = torch.zeros(1, device="cuda")
        dist.barrier(group=group)   # every rank's block is mapped and zeroed before the first frame

    def select(self):
        capi.check(capi.lib().psm_disp_select_keys_p2p(self.de.handle), self.de.handle)

    def barrier(self):
        import torch.distributed as dist
        dist.all_reduce(self._flag, group=self.group)  # stream-ordered cross-rank barrier (device_sync=False only)

    def reduce(self):
        capi.check(capi.lib().psm_disp_reduce_p2p(self.de.handle), self.de.handle)

    def fetch(self, lmap_ptr, rmap_ptr):
        """host maps of the context's format: uint8, or uint16 on a 16-bit context (rows of W elements)"""
        L = capi.lib()
        if _wide(self.de):
            capi.check(L.psm_disp_fetch_p2p_u16(self.de.handle, lmap_ptr, 2 * self.de.wid, rmap_ptr, 2 * self.de.wid),
                       self.de.handle)
        else:
            capi.check(L.psm_disp_fetch_p2p(self.de.handle, lmap_ptr, self.de.wid, rmap_ptr, self.de.wid), self.de.handle)

    def frame(self, lmap_ptr=None, rmap_ptr=None):
        """select -> reduce [-> fetch]; with device_sync=False a barrier follows select and reduce."""
        self.select()
        if not self.device_sync:
            self.barrier()
        self.reduce()
        if not self.device_sync:
            self.barrier()
        if lmap_ptr is not None:
            self.fetch(lmap_ptr, rmap_ptr)


class BandedUpload:
    """N > 1, frames in HOST memory: every rank uploads only its row band of both images over PCIe (H/N rows) and
    the bands are all-gathered over NVLink, so the host->device bytes per rank shrink with N instead of every
    rank uploading both full images.  The gathered interleaved images feed psm_set_images_device.
    upload_async() runs the band copies and the all-gathers on a side stream into the buffer set that is not in
    use; commit() makes the context's stream wait for them and ingests -- frame k+1 uploads while frame k computes."""

    def __init__(self, de, world, rank, dtype="float32", group=None):
        import torch
        if dtype != "float32":
            raise ValueError("BandedUpload gathers float32 frames (psm_set_images_device takes float images)")
        self.de, self.world, self.rank, self.group = de, world, rank, group
        self.r0, self.r1, self.rows = band_rows(de.hei, world, rank)
        W = de.wid
        self.band = [torch.zeros((self.rows, W, 3), dtype=torch.float32, device="cuda") for _ in range(2)]
        self.full = [[torch.empty((world * self.rows, W, 3), dtype=torch.float32, device="cuda") for _ in range(2)]
                     for _ in range(2)]
        self.step_bytes = W * 3 * 4
        self.side = torch.cuda.Stream()
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.consumed = [None, None]
        self.cur, self.pending = 0, None
        bind_to_current_stream(de)   # the ingest kernels run on torch's current stream, which waits for the side stream

    def h2d_bytes(self):
        return 2 * (self.r1 - self.r0) * self.de.wid * 3 * 4

    def upload_async(self, left_pinned, right_pinned):
        """left_pinned / right_pinned: pinned host tensors [H, W, 3] float32 of the FULL frame (each rank reads its band)."""
        import torch
        import torch.distributed as dist
        if self.pending is not None:
            raise RuntimeError("an upload is already pending: call commit() first")
        s = self.cur ^ 1
        with torch.cuda.stream(self.side):
            if self.consumed[s] is not None:
                self.side.wait_event(self.consumed[s])   # the ingest of the frame that last used this set is done
            for k, src in enumerate((left_pinned, right_pinned)):
                self.band[k][: self.r1 - self.r0].copy_(src[self.r0:self.r1], non_blocking=True)
                dist.all_gather_into_tensor(self.full[s][k].view(-1), self.band[k].view(-1), group=self.group)
            self.ready[s].record(self.side)
        self.pending = s

    def commit(self):
        import torch
        if self.pending is None:
            raise RuntimeError("commit() without a pending upload_async()")
        s, self.pending = self.pending, None
        main = torch.cuda.current_stream()
        main.wait_event(self.ready[s])
        capi.check(capi.lib().psm_set_images_device(self.de.handle, self.full[s][0].data_ptr(), self.step_bytes,
                                                    self.full[s][1].data_ptr(), self.step_bytes), self.de.handle)
        ev = torch.cuda.Event()
        ev.record(main)
        self.consumed[s] = ev
        self.cur = s

    def upload(self, left_pinned, right_pinned):
        self.upload_async(left_pinned, right_pinned)
        self.commit()
