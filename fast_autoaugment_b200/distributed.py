"""Multi-GPU use of the hot path (SURVEY.md 8e): one process per GPU, ``torch.distributed``.

Augmentation shards trivially - every op's dependencies are inside one image - so ranks process
their own contiguous shard with no data-path collective.  The only exchange step is **Mixup with
global pairing**, i.e. a permutation over the *global* batch (reference ``aug_mixup.py:13-23`` is
rank-local under DDP, ``train.py:55``; global pairing is an extension):

* the pairing and lambda are derived from a shared seed, identically on every rank (no
  communication);
* every sample's partner is needed by exactly ONE sample (the pairing is a permutation), so the exchange
  is a **partner-only all-to-all** of raw uint8 images (``mixup_global``): a rank receives only the <= B/G
  images its own samples pair with - 1/G of what a whole-pool all-gather would deliver - 3 B/px on the wire:
  half of the fp16 output, a quarter of fp32.
  Mixing is linear, so "augment the partner here" equals "augment there, send, mix";
* the fused-Mixup kernel recomputes each partner's augmentation from the received raw image with the
  partner's own decisions: Philox records drawn for the GLOBAL sample indices on every rank (16 + 8 n_op
  bytes per sample, no communication) and gathered into pool order.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .engine import CompiledPolicy, TailSpec, augment_batch, make_rng


def shard_bounds(n: int, rank: int, world: int):
    """Contiguous shard [lo, hi) of n samples for `rank` (DistributedSampler-style equal shards:
    n must be divisible by world, reference data.py:205-212 pads instead)."""
    if n % world:
        raise ValueError("global batch %d is not divisible by world size %d" % (n, world))
    per = n // world
    return rank * per, (rank + 1) * per


def global_pairing(global_batch: int, alpha: float, seed: int, step: int):
    """(perm, lam) of reference ``mixup`` (aug_mixup.py:14,18-19) for the GLOBAL batch, identical on
    every rank without communication: both draws come from generators seeded with (seed, step)."""
    g = torch.Generator(device="cpu")
    g.manual_seed((int(seed) * 1000003 + int(step)) & 0x7FFFFFFFFFFFFFFF)
    perm = torch.randperm(global_batch, generator=g)
    # (a counter-seeded generator: 8 us to construct; RandomState(seed) costs 100 us of Mersenne-Twister seeding per step)
    rs = np.random.Generator(np.random.PCG64([int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF]))
    lam = rs.beta(alpha, alpha)
    lam = max(lam, 1.0 - lam)
    assert 0.0 <= lam <= 1.0, lam
    return perm, float(lam)


class _PinnedRing:
    """Small CPU index tensors go to the device through pinned staging buffers and ``non_blocking`` copies: a plain
    ``.to(device)`` of pageable memory blocks the host until everything queued on the stream has run, which serialises the
    host's planning of step N+1 with the kernels of step N.  A buffer is reused only after the copy that read it has run."""
    _rings = {}

    @classmethod
    def upload(cls, t: torch.Tensor, device, dtype=None) -> torch.Tensor:
        t = t.contiguous() if dtype is None else t.to(dtype).contiguous()
        n = t.numel()
        out = torch.empty(t.shape, dtype=t.dtype, device=device)
        if n == 0:
            return out
        key = (str(device), t.dtype, 1 << max(6, (n - 1).bit_length()))
        ring = cls._rings.setdefault(key, {"bufs": [], "evs": [], "next": 0})
        if len(ring["bufs"]) < 8:
            ring["bufs"].append(torch.empty(key[2], dtype=t.dtype).pin_memory())
            ring["evs"].append(None)
            i = len(ring["bufs"]) - 1
        else:
            i = ring["next"]; ring["next"] = (i + 1) % 8
            if ring["evs"][i] is not None:
                ring["evs"][i].synchronize()
        buf = ring["bufs"][i][:n]
        buf.copy_(t.reshape(-1))
        out.reshape(-1).copy_(buf, non_blocking=True)
        ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(device))
        ring["evs"][i] = ev
        return out


def gather_pool(local: torch.Tensor, group=None) -> torch.Tensor:
    """All-gather equal-sized shards along dim 0 (NCCL on CUDA tensors, gloo on CPU tensors)."""
    world = dist.get_world_size(group)
    local = local.contiguous()
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    if local.is_cuda:
        dist.all_gather_into_tensor(out, local, group=group)
    else:
        dist.all_gather(list(out.chunk(world, 0)), local, group=group)
    return out


def partner_plan(perm: torch.Tensor, rank: int, world: int):
    """The partner-only exchange for the global pairing ``perm`` (contiguous equal shards), computed locally on
    every rank.  Returns ``(send_idx, send_counts, recv_counts, partner_pool, recv_global)``:

    * ``send_idx``     local indices of the images this rank sends, grouped by destination rank (within a
      group in the order of the destination's samples), ``send_counts[r]`` of them go to rank r;
    * ``recv_counts``  how many images arrive from each rank; they land, grouped by source rank, behind the
      local shard in the pool ``[local shard | received]``;
    * ``partner_pool`` for every local sample the pool index of its partner (a local index when the partner is
      in this rank's own shard - nothing is sent to oneself);
    * ``recv_global``  the global sample index of every received image (for its decision records)."""
    n = int(perm.numel())
    b = n // world
    perm = perm.to(torch.int64).cpu()
    if world == 1:                                              # every partner is local: nothing is sent
        e = torch.empty(0, dtype=torch.int64)
        return e, [0], [0], perm.clone(), e
    owner = perm // b                                           # rank that owns each sample's partner
    lo = rank * b
    send_idx, send_counts = [], []
    for r in range(world):                                      # what rank r's samples need from my shard
        pr = perm[r * b:(r + 1) * b]
        mine = pr[(owner[r * b:(r + 1) * b] == rank)] if r != rank else pr[:0]
        send_idx.append(mine - lo)
        send_counts.append(int(mine.numel()))
    my_p, my_owner = perm[lo:lo + b], owner[lo:lo + b]
    partner_pool = torch.empty(b, dtype=torch.int64)
    recv_counts, recv_global = [], []
    base = b
    for s in range(world):                                      # received block of source rank s: my samples in order
        sel = (my_owner == s).nonzero(as_tuple=True)[0]
        if s == rank:
            partner_pool[sel] = my_p[sel] - lo
            recv_counts.append(0)
            continue
        partner_pool[sel] = base + torch.arange(sel.numel(), dtype=torch.int64)
        recv_counts.append(int(sel.numel()))
        recv_global.append(my_p[sel])
        base += int(sel.numel())
    return (torch.cat(send_idx) if send_idx else torch.empty(0, dtype=torch.int64), send_counts, recv_counts,
            partner_pool, torch.cat(recv_global) if recv_global else torch.empty(0, dtype=torch.int64))


def exchange_partners(local: torch.Tensor, send_idx, send_counts, recv_counts, group=None) -> torch.Tensor:
    """All-to-all of the planned rows of ``local`` (dim 0); returns the received rows grouped by source rank."""
    send = local.index_select(0, send_idx.to(local.device))
    out = torch.empty((sum(recv_counts),) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_to_all_single(out, send, output_split_sizes=list(recv_counts), input_split_sizes=list(send_counts), group=group)
    return out


def philox_records(policy: CompiledPolicy, n: int, h: int, w: int, tail: TailSpec, seed: int, first_index: int, device):
    """Decision records of samples [first_index, first_index + n) drawn by the device sampler: uint8 tensors
    ``(samples [n,16], boxes [n, 8*n_op])`` - what the fused Philox path would use for those indices."""
    t = tail.c_struct(h, w)
    rng = make_rng(seed, first_index, tail)
    d_s = torch.zeros((n, 16), dtype=torch.uint8, device=device)
    d_b = torch.zeros((n, 8 * policy.n_op), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib.faa_sample_philox(policy.handle, n, h, w, C.byref(t), C.byref(rng), d_s.data_ptr(), d_b.data_ptr(),
                                              C.c_void_p(torch.cuda.current_stream(device).cuda_stream)))
    return d_s, d_b


def mix_augmented(policy: CompiledPolicy, a_u8: torch.Tensor, pool_u8: torch.Tensor, partner_pool: torch.Tensor, tail: TailSpec,
                  lam: float, zero_box_a=None, zero_box_pool=None, out=None):
    """``norm(a[i]) * lam + norm(pool[partner_pool[i]]) * (1 - lam)`` for AUGMENTED uint8 HWC images (C ABI ``faa_mix_u8``):
    ToTensor + Normalize + CutoutDefault boxes (int16 [n,4] CUDA tensors, half-open y0,y1,x0,x1) + aug_mixup.py:21."""
    b, h, w, _ = a_u8.shape
    t = tail.c_struct(h, w)
    if out is None:
        out = torch.empty((b, 3, h, w), dtype=tail.out_dtype, device=a_u8.device)
    part = partner_pool if (partner_pool.is_cuda and partner_pool.dtype == torch.int32) else \
        _PinnedRing.upload(partner_pool.cpu(), a_u8.device, torch.int32)
    za = zero_box_a.contiguous() if zero_box_a is not None else None
    zp = zero_box_pool.contiguous() if zero_box_pool is not None else None
    with torch.cuda.device(a_u8.device):
        _lib.check(_lib.lib.faa_mix_u8(policy.handle, a_u8.data_ptr(), pool_u8.data_ptr(), part.data_ptr(),
                                       za.data_ptr() if za is not None else None, zp.data_ptr() if zp is not None else None,
                                       out.data_ptr(), b, h, w, C.byref(t), float(np.float32(lam)), float(np.float32(1 - lam)),
                                       C.c_void_p(torch.cuda.current_stream(a_u8.device).cuda_stream)))
    return out


def mixup_global(policy: CompiledPolicy, local_u8: torch.Tensor, targets: torch.Tensor, tail: TailSpec, alpha: float,
                 seed: int, step: int, group=None, timing=None):
    """Augment this rank's shard and mix every sample with its partner from the GLOBAL batch (module doc):

    1. the shard is augmented ONCE, to uint8 HWC (policy + RandomCrop + HFlip; decisions = Philox keyed by the global
       sample index);
    2. partner-only all-to-all of the AUGMENTED uint8 images (3 B/px; a rank receives only what its samples pair with);
    3. one streaming pass (``faa_mix_u8``) normalises both sources, applies each source's CutoutDefault box and mixes in fp32.

    Returns ``(data, targets, partner_targets, lam)`` like reference ``mixup`` (aug_mixup.py:23); the values equal the
    fused single-GPU launch ``augment_batch(..., partner=perm, lam=lam)`` on the global batch.  ``timing``: optional dict,
    receives CUDA events ``ex0``/``ex1`` around the exchange and ``recv_bytes``."""
    rank, world = (dist.get_rank(group), dist.get_world_size(group)) if dist.is_initialized() else (0, 1)
    b, h, w = local_u8.shape[0], local_u8.shape[1], local_u8.shape[2]
    n = b * world
    dev = local_u8.device
    perm, lam = global_pairing(n, alpha, seed, step)
    lo, _ = shard_bounds(n, rank, world)
    send_idx, send_counts, recv_counts, partner_pool, recv_global = partner_plan(perm, rank, world)
    # the plan goes to the device BEFORE any kernel of this step is queued (asynchronous copies from pinned staging)
    partner_dev = _PinnedRing.upload(partner_pool, dev, torch.int32)
    send_dev = _PinnedRing.upload(send_idx, dev) if world > 1 else None
    tgt_idx_dev = _PinnedRing.upload(perm[lo:lo + b], dev)
    # 1. this shard, augmented to uint8 (the CutoutDefault box acts on the normalised tensor: step 3)
    u8_tail = TailSpec(tail.out_size, tail.crop_pad, tail.hflip, tail.mean, tail.std, 0, torch.uint8)
    rng = make_rng(seed, step * n + lo, tail)
    rng.zero_box_len = 0                                         # (its Philox block is separate: the other draws do not move)
    oh, ow = tail.out_size if tail.out_size is not None else (h, w)
    n_recv = sum(recv_counts)
    pool = torch.empty((b + n_recv, oh, ow, 3), dtype=torch.uint8, device=dev)      # [own augmented shard | received partners]
    if timing is not None:
        timing["a0"] = torch.cuda.Event(enable_timing=True); timing["a0"].record()
    aug = augment_batch(policy, local_u8, u8_tail, rng=rng, out=pool[:b])
    # 2. partners: straight into the tail of the pool
    if timing is not None:
        timing["ex0"] = torch.cuda.Event(enable_timing=True); timing["ex0"].record()
    if world > 1:
        send = aug.index_select(0, send_dev)
        dist.all_to_all_single(pool[b:], send, output_split_sizes=list(recv_counts), input_split_sizes=list(send_counts), group=group)
    all_targets = gather_pool(targets, group) if world > 1 else targets
    if timing is not None:
        timing["ex1"] = torch.cuda.Event(enable_timing=True); timing["ex1"].record()
        timing["recv_bytes"] = int(n_recv) * oh * ow * 3
    # 3. zero boxes of every source (decisions are a function of the global index: no communication), then the mix
    za = zp = None
    if tail.cutout > 0:
        rec_s, _ = philox_records(policy, n, h, w, tail, seed, step * n, dev)
        zb_all = rec_s[:, 8:16].contiguous().view(torch.int16)                      # faa_sample_t.zero_box
        ids = _PinnedRing.upload(torch.cat([torch.arange(lo, lo + b, dtype=torch.int64), recv_global]), dev)
        zp = zb_all.index_select(0, ids)
        za = zp[:b]
    if timing is not None:
        timing["m0"] = torch.cuda.Event(enable_timing=True); timing["m0"].record()
    data = mix_augmented(policy, aug, pool, partner_dev, tail, lam, za, zp)
    if timing is not None:
        timing["m1"] = torch.cuda.Event(enable_timing=True); timing["m1"].record()
    return data, targets, (all_targets[tgt_idx_dev] if all_targets.is_cuda else all_targets[perm[lo:lo + b]]), lam


JPEG_INDEX_CHUNK = 16 << 20                    # bytes of each rank's delta per all-gather round of share_jpeg_index


def _pack_delta(paths, lengths, first, points):
    """a ``JpegIndex.delta`` as one uint8 array: int64 [files, path bytes, points], the file lengths, the path lengths
    and the point offsets (int64 each), the points (16 bytes each), then the paths back to back.  A delta of no file
    packs to no bytes."""
    if not len(paths):
        return np.zeros(0, np.uint8)
    plen = np.array([len(p) for p in paths], np.int64)
    head = np.array([len(paths), int(plen.sum()), len(points)], np.int64)
    return np.concatenate([head.view(np.uint8), np.ascontiguousarray(lengths, np.int64).view(np.uint8),
                           plen.view(np.uint8), np.ascontiguousarray(first, np.int64).view(np.uint8),
                           np.ascontiguousarray(points).view(np.uint8).reshape(-1),
                           np.frombuffer(b"".join(bytes(p) for p in paths), np.uint8)])


def _unpack_delta(buf):
    """``_pack_delta``'s ``(paths, lengths, first, points)`` of ``buf``; ValueError when its sizes do not add up"""
    if buf.size < 24:
        raise ValueError("%d bytes, shorter than its header" % buf.size)
    n, nb, npt = (int(v) for v in np.frombuffer(buf, np.int64, 3))
    if min(n, nb, npt) < 0 or buf.size != 24 + 8 * (3 * n + 1) + _lib.JPEG_SYNC_DTYPE.itemsize * npt + nb:
        raise ValueError("%d bytes do not hold %d files, %d path bytes and %d points" % (buf.size, n, nb, npt))
    ints = np.frombuffer(buf, np.int64, 3 * n + 1, 24)
    lengths, plen, first = ints[:n], ints[n:2 * n], ints[2 * n:]
    at = 24 + 8 * (3 * n + 1)
    points = np.frombuffer(buf, _lib.JPEG_SYNC_DTYPE, npt, at)
    names = buf[at + points.nbytes:].tobytes()
    if (plen < 0).any() or int(plen.sum()) != nb:
        raise ValueError("path lengths do not add up to %d bytes" % nb)
    ends = np.cumsum(plen).tolist()
    return [names[e - k:e] for e, k in zip(ends, plen.tolist())], lengths, first, points


def _fail_everywhere(err, group, what="JPEG index exchange"):
    """called on every rank at once when the flags of a collective step showed a failure: raise on every rank, naming
    each rank's error"""
    msgs = [None] * dist.get_world_size(group)
    dist.all_gather_object(msgs, None if err is None else "%s: %s" % (type(err).__name__, err), group=group)
    raise RuntimeError("%s failed: " % what + "; ".join(
        "rank %d: %s" % (r, m) for r, m in enumerate(msgs) if m is not None)) from err


def _exchange_device(group):
    """where the exchanges' tensors live: the current device under NCCL, the host otherwise"""
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")


def _gather_sizes(mine, err, dev, group, what):
    """all-gather of every rank's byte count (-1: the rank has nothing to send, ``err`` says why); raises on every rank
    when any rank failed"""
    sizes = gather_pool(torch.tensor([-1 if mine is None else mine.size], dtype=torch.int64, device=dev), group)
    sizes = sizes.cpu().tolist()
    if min(sizes) < 0:
        _fail_everywhere(err, group, what)
    return sizes


def _gather_rounds(mine, sizes, err, dev, group, chunk_bytes):
    """every rank's uint8 array ``mine`` (of ``sizes[rank]`` bytes) to every rank, in all-gather rounds of at most
    ``chunk_bytes`` per rank: (arrays in rank order, own one included, error).  Every rank enters every round whatever
    fails locally; a failure is returned, not raised."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    top = max(sizes)
    step = max(1, min(int(chunk_bytes), top))
    bufs = None
    try:
        bufs = [mine if r == rank else np.empty(sizes[r], np.uint8) for r in range(world)]
    except Exception as e:                                       # noqa: BLE001
        err = e
    for at in range(0, top, step):
        m = min(step, top - at)
        send = torch.zeros(m, dtype=torch.uint8)
        send[:max(0, min(m, sizes[rank] - at))] = torch.from_numpy(mine[at:at + m])
        got = gather_pool(send.to(dev), group).cpu().numpy()
        if err is None:
            try:
                for r in range(world):
                    k = min(m, sizes[r] - at)
                    if r != rank and k > 0:
                        bufs[r][at:at + k] = got[r * m:r * m + k]
            except Exception as e:                               # noqa: BLE001
                err = e
    return bufs, err


def agree(err, group=None, what="collective step"):
    """Collective: all-gather of every rank's success; when any rank failed (``err`` not None there), RuntimeError on
    every rank naming each rank's error"""
    oks = gather_pool(torch.tensor([int(err is None)], dtype=torch.int64, device=_exchange_device(group)), group)
    if not bool(oks.all()):
        _fail_everywhere(err, group, what)


def share_jpeg_index(index, group=None, chunk_bytes=JPEG_INDEX_CHUNK):
    """Collective: every rank of ``group`` sends the entries its ``JpegIndex`` learned since the last exchange
    (``index.delta()``) to every other rank, and enters the other ranks' deltas in rank order (``index.merge``), so
    every rank's index ends up listing what any rank learned.  Returns the number of entries merged here.

    One all-gather of the packed deltas' sizes, then, when any is not empty, rounds of all-gathers of at most
    ``chunk_bytes`` of every rank's delta (so no rank ever holds world x its delta in flight), then one all-gather of
    success flags.  Device tensors on the current device with NCCL, host tensors otherwise.  Every rank enters the
    same collectives whatever fails locally: a delta that cannot be packed, one that does not unpack or merge (the
    same verdict on every rank that reads it) or any other local error raises RuntimeError on every rank, naming each
    rank's error, instead of leaving the others waiting.  Entries merged before a failure stay (a point only decides
    how a file's decode is split, never its pixels)."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    dev = _exchange_device(group)
    err = mine = None
    try:
        mine = _pack_delta(*index.delta())
    except Exception as e:                                       # noqa: BLE001
        err = e
    sizes = _gather_sizes(mine, err, dev, group, "JPEG index exchange")
    if max(sizes) == 0:
        return 0
    bufs, err = _gather_rounds(mine, sizes, err, dev, group, chunk_bytes)
    merged = 0
    if err is None:
        try:
            for r in range(world):
                if r == rank or sizes[r] == 0:
                    continue
                try:
                    delta = _unpack_delta(bufs[r])
                    index.merge(*delta)
                except ValueError as e:
                    raise ValueError("rank %d's JPEG index delta is malformed: %s" % (r, e)) from e
                merged += len(delta[0])
        except Exception as e:                                   # noqa: BLE001
            err = e
    agree(err, group, "JPEG index exchange")
    return merged


def local_ranks(hosts, rank):
    """the ranks whose host name (``hosts``, one per rank) is ``rank``'s, in rank order"""
    return [r for r, h in enumerate(hosts) if h == hosts[rank]]


def host_ranks(group=None):
    """Collective: all-gathers ``socket.gethostname()`` and returns ``local_ranks`` of this rank"""
    import socket
    hosts = [None] * dist.get_world_size(group)
    dist.all_gather_object(hosts, socket.gethostname(), group=group)
    return local_ranks(hosts, dist.get_rank(group))


def fit_error(needs, frees):
    """the RuntimeError message when any rank's need (bytes) exceeds its free device memory, else None"""
    if all(n <= f for n, f in zip(needs, frees)):
        return None
    return "the resident JPEG store does not fit: " + "; ".join(
        "rank %d needs %d bytes, %d free%s" % (r, n, f, " (too little)" if n > f else "")
        for r, (n, f) in enumerate(zip(needs, frees)))


def check_fit(need, free, err=None, group=None):
    """Collective: every rank's device-memory need and free bytes (``need`` None: the rank failed before it knew,
    ``err`` says why).  RuntimeError on every rank when any rank failed or any shard does not fit (``fit_error``)."""
    dev = _exchange_device(group)
    got = gather_pool(torch.tensor([-1 if need is None else int(need), int(free)], dtype=torch.int64, device=dev)
                      .view(1, 2), group).cpu().tolist()
    if min(n for n, _ in got) < 0:
        _fail_everywhere(err, group, "resident JPEG store")
    msg = fit_error([n for n, _ in got], [f for _, f in got])
    if msg is not None:
        raise RuntimeError(msg)


def gather_bytes(mine, err=None, group=None, chunk_bytes=JPEG_INDEX_CHUNK, what="resident JPEG store"):
    """Collective: every rank's uint8 array ``mine`` (None when the rank failed to make it, ``err`` then its error) to
    every rank, in ``share_jpeg_index``'s rounds.  Returns ``(arrays in rank order, error)``; the caller reads them and
    ends with ``agree``.  Raises on every rank when any rank had nothing to send."""
    dev = _exchange_device(group)
    sizes = _gather_sizes(mine, err, dev, group, what)
    if max(sizes) == 0:
        return [np.zeros(0, np.uint8) for _ in sizes], err
    return _gather_rounds(mine, sizes, err, dev, group, chunk_bytes)


class _RawCuda:
    """zero-copy torch view of a raw device allocation (``__cuda_array_interface__``)"""
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "|u1", "data": (int(ptr), False), "version": 3, "strides": None}


class PeerPool:
    """Per-rank uint8 buffers ``[slots][b][H][W][3]`` that EVERY rank of the node can read: each rank allocates its own
    (C ABI ``faa_peer_alloc``: cudaMalloc + cudaIpcGetMemHandle), the 64-byte handles are all-gathered and every rank maps
    its peers' buffers under ITS device (``faa_peer_open``: cudaIpcOpenMemHandle with lazy peer access), so that its kernels
    can dereference them over NVLink.  ``ptr(rank, slot)`` is the device address of that rank's buffer in THIS process."""

    def __init__(self, b: int, h: int, w: int, device, group=None, slots: int = 2):
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.b, self.h, self.w, self.slots = b, h, w, slots
        self.img_bytes = h * w * 3
        self.device = torch.device(device)
        nbytes = slots * b * self.img_bytes
        # every rank runs the SAME sequence of collectives whether or not its local CUDA calls succeed, so that a failure on
        # one rank becomes an exception on all of them (and the caller's fallback) instead of a hang
        self._own, self._opened, self.base, self.local = 0, [], [], None
        err, hb = None, None
        try:
            with torch.cuda.device(self.device):
                ptr, handle = C.c_void_p(), (C.c_ubyte * 64)()
                _lib.check(_lib.lib.faa_peer_alloc(nbytes, C.byref(ptr), handle))
                self._own, hb = ptr.value, bytes(handle)
                self.local = torch.as_tensor(_RawCuda(self._own, (slots, b, h, w, 3)), device=self.device)
        except Exception as e:                                   # noqa: BLE001
            err = e
        gathered = [None] * self.world
        dist.all_gather_object(gathered, (self.device.index, hb), group=group)
        if err is None and all(g[1] is not None for g in gathered):
            try:
                with torch.cuda.device(self.device):
                    for r in range(self.world):
                        if r == self.rank:
                            self.base.append(self._own)
                            continue
                        peer_dev, peer_hb = gathered[r]
                        _lib.check(_lib.lib.faa_enable_peer_access(int(peer_dev)))
                        p = C.c_void_p()
                        _lib.check(_lib.lib.faa_peer_open((C.c_ubyte * 64).from_buffer_copy(peer_hb), C.byref(p)))
                        self.base.append(p.value)
                        self._opened.append(p.value)
                    self.flag = torch.zeros(1, dtype=torch.int32, device=self.device)
                    torch.cuda.synchronize(self.device)
            except Exception as e:                               # noqa: BLE001
                err = e
        elif err is None:
            err = RuntimeError("a peer could not allocate its exportable buffer")
        oks = [None] * self.world
        dist.all_gather_object(oks, err is None, group=group)         # (also the barrier: every mapping exists)
        if not all(oks):
            self._release(group)
            raise RuntimeError("peer pool unavailable on rank(s) %s%s" % (
                [r for r, ok in enumerate(oks) if not ok], ": %s" % err if err is not None else ""))

    def _release(self, group=None):
        for p in self._opened:
            _lib.lib.faa_peer_close(C.c_void_p(p))
        self._opened = []
        dist.barrier(group=group)                                # nobody maps our buffer any more
        if self._own:
            self.local = None
            _lib.lib.faa_peer_free(C.c_void_p(self._own))
            self._own = 0

    def ptr(self, rank: int, slot: int) -> int:
        return self.base[rank] + slot * self.b * self.img_bytes

    def close(self, group=None):
        """unmap the peers' buffers, then (after a barrier: nobody maps ours any more) free our own"""
        torch.cuda.synchronize(self.device)
        with torch.cuda.device(self.device):
            self._release(group)


def partner_pointers(perm: torch.Tensor, rank: int, world: int, bases, img_bytes: int) -> torch.Tensor:
    """Address of every local sample's partner image for the pairing ``perm`` (contiguous equal shards): sample i of rank
    ``rank`` pairs with global sample ``p = perm[rank * b + i]``, which is image ``p % b`` of rank ``p // b``, whose buffer
    starts at ``bases[p // b]`` (as mapped in THIS process).  int64 tensor [b]; host logic only."""
    n = int(perm.numel())
    b = n // world
    mine = perm[rank * b:(rank + 1) * b].to(torch.int64).cpu()
    base = torch.tensor([int(x) for x in bases], dtype=torch.int64)
    return base[mine // b] + (mine % b) * int(img_bytes)


def mixup_global_peer(policy: CompiledPolicy, local_u8: torch.Tensor, targets: torch.Tensor, tail: TailSpec, alpha: float,
                      seed: int, step: int, pool: PeerPool, group=None, timing=None):
    """``mixup_global`` with the exchange fused into the mix kernel: every rank augments its shard into its slot of the
    ``PeerPool``, ONE tiny all-reduce orders the ranks (partners' images complete), and ``faa_mix_u8_peer`` reads each
    partner image straight from its owner's memory over NVLink - no all-to-all, no received copy.  Slot ``step % 2``: the
    barrier of step N+1 also tells every rank that its peers are done reading the slot of step N.  Same values as
    ``mixup_global``."""
    rank, world = pool.rank, pool.world
    b, h, w = local_u8.shape[0], local_u8.shape[1], local_u8.shape[2]
    assert (b, h, w) == (pool.b, pool.h, pool.w)
    n = b * world
    dev = local_u8.device
    perm, lam = global_pairing(n, alpha, seed, step)
    lo, _ = shard_bounds(n, rank, world)
    slot = step % pool.slots
    mine = perm[lo:lo + b].to(torch.int64)
    ptrs = partner_pointers(perm, rank, world, [pool.ptr(r, slot) for r in range(world)], pool.img_bytes)
    ptrs_dev = _PinnedRing.upload(ptrs, dev)
    tgt_idx_dev = _PinnedRing.upload(mine, dev)
    u8_tail = TailSpec(tail.out_size, tail.crop_pad, tail.hflip, tail.mean, tail.std, 0, torch.uint8)
    rng = make_rng(seed, step * n + lo, tail)
    rng.zero_box_len = 0
    if timing is not None:
        timing["a0"] = torch.cuda.Event(enable_timing=True); timing["a0"].record()
    aug = augment_batch(policy, local_u8, u8_tail, rng=rng, out=pool.local[slot])
    if timing is not None:
        timing["ex0"] = torch.cuda.Event(enable_timing=True); timing["ex0"].record()
    if world > 1:
        dist.all_reduce(pool.flag, group=group)                  # every rank's augmentation of this step has run
    all_targets = gather_pool(targets, group) if world > 1 else targets
    if timing is not None:
        timing["ex1"] = torch.cuda.Event(enable_timing=True); timing["ex1"].record()
        timing["recv_bytes"] = int((mine // b != rank).sum()) * pool.img_bytes
    za = zp = None
    if tail.cutout > 0:
        rec_s, _ = philox_records(policy, n, h, w, tail, seed, step * n, dev)
        zb_all = rec_s[:, 8:16].contiguous().view(torch.int16)
        za = zb_all[lo:lo + b].contiguous()
        zp = zb_all.index_select(0, tgt_idx_dev)
    t = tail.c_struct(h, w)
    out = torch.empty((b, 3, h, w), dtype=tail.out_dtype, device=dev)
    if timing is not None:
        timing["m0"] = torch.cuda.Event(enable_timing=True); timing["m0"].record()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib.faa_mix_u8_peer(policy.handle, aug.data_ptr(), ptrs_dev.data_ptr(),
                                            za.data_ptr() if za is not None else None, zp.data_ptr() if zp is not None else None,
                                            out.data_ptr(), b, h, w, C.byref(t), float(np.float32(lam)), float(np.float32(1 - lam)),
                                            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    if timing is not None:
        timing["m1"] = torch.cuda.Event(enable_timing=True); timing["m1"].record()
    return out, targets, all_targets[tgt_idx_dev], lam

