"""Multi-GPU: x-slab decomposition of the particle set, one process per GPU (torch.distributed).

Why slabs: the cell index is x-major (CUDAFunctions.cuh:68), so an x-slab of cells is one contiguous key
range and, after the sort, one contiguous particle range; the interaction range is one cell
(cellLength >= radius, main.cpp:57), so the halo is ONE plane of cells per side (SURVEY 8e).

Rank g owns global cell planes [X_g, X_{g+1}).  Its libsphk context covers the local grid
[X_g - 1, X_{g+1} + 1) (sphk_grid.origin), and its fluid arrays hold, sorted by local cell index,

        [ ghost-left (plane X_g - 1) | owned | ghost-right (plane X_{g+1}) ]

Per step (`SlabSystem.begin_step`) -- ONE exchange and ONE search:
  1. every rank sends its two outermost owned planes per side (contiguous slices of last step's sorted order; a
     particle moves less than one plane per step, so these are all particles that can now be in the neighbour's
     last owned plane or in its ghost plane) -- count first, then one packed message per neighbour;
  2. it searches [candidates-from-left | own particles | candidates-from-right] once.  The sort itself decides
     everything: local plane 0 / w+1 = ghosts (own particles that left the slab included), planes 1..w = owned
     (immigrants included), keys outside the local grid = candidates that belong to neither -> sorted to the end
     and ignored (no cell range contains them).  Ownership is decided by the global cell plane on both sides, so
     no particle is lost or duplicated;
  3. sweeps are restricted to the owned range (sphk_set_active_range).
During the solver step every field a sweep reads from neighbours and a previous sweep changed is refreshed
on the ghosts: the owner's first/last plane slice of the API array is sent to the neighbour's ghost slice
(contiguous -> no packing kernels), then sphk_push_range mirrors it into the packed records.

Collectives: point-to-point send/recv with the two x-neighbours only (NCCL over NVLink; gloo in the CPU
tests); a 1-float all-reduce only in adaptive-iteration DFSPH.  All three solvers shard (PBD additionally
refreshes the ghosts' positions after every projection).  Particle order inside a cell differs from a
single-GPU run (immigrants are appended), so sums are formed in a different order: multi-GPU parity is
<= 1e-5 like every floating-point check here, not bit-exact.

`SlabExchange` (pure torch + torch.distributed, device-agnostic) is what the gloo tests exercise.
"""
from __future__ import annotations

import ctypes as C
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

from . import capi
from .capi import SphkGrid, check
from . import scene as scene_mod
from .engine import EPSILON, ParticleSet, SphkOps, _ptr, device_boundary_shell, device_fluid_block


def choose_cuts_weighted(plane_of_column: np.ndarray, weight: int, n_planes: int, world: int) -> list[int]:
    """choose_cuts for a lattice given by its columns: every column carries `weight` particles."""
    counts = np.bincount(plane_of_column, minlength=n_planes).astype(np.int64) * int(weight)
    return _cuts_from_counts(counts, n_planes, world)


def choose_cuts(plane_of_particle: np.ndarray, n_planes: int, world: int) -> list[int]:
    """Plane indices X_0=0 < X_1 < ... < X_world=n_planes that balance the particle counts (the CDF along x is
    free: cellStart[x*cy*cz], SURVEY 8e).  Every slab gets at least one plane."""
    counts = np.bincount(plane_of_particle, minlength=n_planes).astype(np.int64)
    return _cuts_from_counts(counts, n_planes, world)


def skew_cuts(cuts: list[int], skew: int, n_planes: int) -> list[int]:
    world = len(cuts) - 1
    out = list(cuts)
    for g in range(1, world):
        out[g] = min(max(cuts[g] + skew, out[g - 1] + 1), n_planes - (world - g))
    return out


def _cuts_from_counts(counts: np.ndarray, n_planes: int, world: int) -> list[int]:
    cdf = np.cumsum(counts)
    total = int(cdf[-1])
    cuts = [0]
    for g in range(1, world):
        x = int(np.searchsorted(cdf, total * g / world, side="left")) + 1
        x = max(x, cuts[-1] + 1)
        x = min(x, n_planes - (world - g))
        cuts.append(x)
    cuts.append(n_planes)
    return cuts


class SlabExchange:
    """Neighbour exchange along the slab axis.  All tensors live on `device` (cuda for NCCL, cpu for gloo)."""

    def __init__(self, rank: int, world: int, device, group=None):
        self.rank, self.world, self.device, self.group = rank, world, torch.device(device), group
        self.left = rank - 1 if rank > 0 else None
        self.right = rank + 1 if rank < world - 1 else None
        self.bytes_sent = 0
        self.messages = 0
        # gloo cannot move CUDA tensors: stage through the host (single-GPU test boxes run 2 ranks on one GPU)
        self.stage = self.device.type == "cuda" and dist.get_backend(group) == "gloo"

    def _run(self, ops):
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()

    def _p2p(self, sends, recvs):
        """sends / recvs: lists of (tensor, peer).  Host-staged when the backend cannot carry device memory."""
        if not self.stage:
            self._run([dist.P2POp(dist.isend, t, p, self.group) for t, p in sends] +
                      [dist.P2POp(dist.irecv, t, p, self.group) for t, p in recvs])
            return
        hs = [(t.detach().cpu().contiguous(), p) for t, p in sends]
        hr = [(torch.empty(t.shape, dtype=t.dtype), p, t) for t, p in recvs]
        self._run([dist.P2POp(dist.isend, t, p, self.group) for t, p in hs] +
                  [dist.P2POp(dist.irecv, h, p, self.group) for h, p, _ in hr])
        for h, _, t in hr:
            t.copy_(h)

    def exchange_counts(self, n_left: int, n_right: int) -> tuple[int, int]:
        """Tell each neighbour how many rows it will receive; returns (from_left, from_right)."""
        send = torch.tensor([n_left, n_right], dtype=torch.int64, device=self.device)
        recv = torch.zeros(2, dtype=torch.int64, device=self.device)
        sends, recvs = [], []
        if self.left is not None:
            sends.append((send[0:1], self.left)); recvs.append((recv[0:1], self.left))
        if self.right is not None:
            sends.append((send[1:2], self.right)); recvs.append((recv[1:2], self.right))
        self._p2p(sends, recvs)
        r = recv.cpu()
        return int(r[0]), int(r[1])

    def exchange(self, to_left: torch.Tensor | None, to_right: torch.Tensor | None, from_left: torch.Tensor | None,
                 from_right: torch.Tensor | None):
        """Sizes are known on both sides.  Buffers must be contiguous; empty messages are skipped."""
        sends, recvs = [], []
        if self.left is not None:
            if to_left is not None and to_left.numel():
                sends.append((to_left, self.left))
                self.bytes_sent += to_left.numel() * to_left.element_size(); self.messages += 1
            if from_left is not None and from_left.numel():
                recvs.append((from_left, self.left))
        if self.right is not None:
            if to_right is not None and to_right.numel():
                sends.append((to_right, self.right))
                self.bytes_sent += to_right.numel() * to_right.element_size(); self.messages += 1
            if from_right is not None and from_right.numel():
                recvs.append((from_right, self.right))
        self._p2p(sends, recvs)

    def all_gather(self, block: torch.Tensor) -> torch.Tensor:
        """Every rank's `block` (same size everywhere), concatenated in rank order."""
        send = block.detach().cpu().contiguous() if self.stage else block.contiguous()
        parts = [torch.empty_like(send) for _ in range(self.world)]
        dist.all_gather(parts, send, group=self.group)
        self.bytes_sent += send.numel() * send.element_size(); self.messages += 1
        return torch.cat(parts).to(block.device)

    def exchange_rows(self, to_left: torch.Tensor, to_right: torch.Tensor):
        """Variable-size row exchange: counts first, then the rows.  Returns (rows_from_left, rows_from_right)."""
        nl, nr = self.exchange_counts(to_left.shape[0] if self.left is not None else 0,
                                      to_right.shape[0] if self.right is not None else 0)
        width = to_left.shape[1]
        fl = torch.empty((nl, width), dtype=to_left.dtype, device=self.device)
        fr = torch.empty((nr, width), dtype=to_left.dtype, device=self.device)
        self.exchange(to_left.contiguous(), to_right.contiguous(), fl, fr)
        return fl, fr


# ---- strays: owned particles that crossed two or more planes since the last sort (include/sphk.h, "Strays") ----------------
# The candidate exchange below covers one plane of motion per step.  The reference's own DFSPH benchmark setting (4 + 4 fixed
# iterations, dt = 0.004) shoots a few hundred particles across tens of planes once the block hits the floor (around step 40
# of the dam break: tools/plane_skip_probe.py), so such particles are taken out of the regular flow and sent to EVERY rank:
# collect (rows into a fixed-size block, position out of the world) -> all-gather -> append behind the assembled set, the
# same sequence on every rank.  The next sort keeps a stray where it landed and drops it everywhere else.
STRAY_HEADER = 4                  # floats in front of the rows: {int32 count, 3 x pad}
OUT_OF_WORLD = -1.0e6


def stray_block_floats(capacity: int, widths) -> int:
    return STRAY_HEADER + capacity * int(sum(widths))


def _widths(arrays):
    return [1 if a.dim() == 1 else int(a.shape[1]) for a in arrays]


def collect_strays_host(arrays, own: tuple, plane_sorted, plane_now, capacity: int) -> torch.Tensor:
    """torch statement of sphk_strays_collect (what the kernel does; the CPU tests run on it): plane_sorted / plane_now are
    the x-plane a slot of the owned range was sorted into and the plane of its position now.  Returns the block."""
    widths = _widths(arrays)
    stride = sum(widths)
    block = torch.zeros(stray_block_floats(capacity, widths), dtype=torch.float32, device=arrays[0].device)
    idx = torch.nonzero((torch.as_tensor(plane_now) - torch.as_tensor(plane_sorted)).abs() >= 2).flatten() + own[0]
    block[:1].view(torch.int32)[0] = int(idx.numel())
    idx = idx[:capacity]
    if idx.numel():
        rows = torch.cat([a[idx].reshape(idx.numel(), w_) for a, w_ in zip(arrays, widths)], 1)
        block[STRAY_HEADER:STRAY_HEADER + rows.numel()] = rows.flatten()
        arrays[0][idx] = OUT_OF_WORLD
    return block


def append_strays_host(gathered: torch.Tensor, world: int, capacity: int, arrays, dst_begin: int) -> int:
    """torch statement of sphk_strays_append: world * capacity slots from dst_begin on.  Returns that slot count."""
    widths = _widths(arrays)
    stride = sum(widths)
    blocks = gathered.reshape(world, stray_block_floats(capacity, widths))
    counts = blocks[:, :1].contiguous().view(torch.int32).flatten().clamp(max=capacity)
    rows = blocks[:, STRAY_HEADER:].reshape(world, capacity, stride).clone()
    unused = torch.arange(capacity, device=gathered.device)[None, :] >= counts[:, None]
    rows[unused] = 0.0
    rows[..., :3][unused] = OUT_OF_WORLD
    rows = rows.reshape(world * capacity, stride)
    c = 0
    for a, w_ in zip(arrays, widths):
        a[dst_begin:dst_begin + world * capacity] = rows[:, c:c + w_].reshape((world * capacity,) + tuple(a.shape[1:]))
        c += w_
    return world * capacity


def exchange_candidates(ex: SlabExchange, arrays, alt, own: tuple, to_left: tuple, to_right: tuple) -> int:
    """Step 1 of the module docstring + the concatenation for step 2.

    arrays    list of per-particle tensors (first dimension = slot); alt: same-shaped scratch set
    own       (begin, end): slots of the particles this rank owned at the end of the last step (sorted order)
    to_left   (begin, end) inside `own`: its first two owned planes;  to_right: its last two owned planes
    Returns n_all; afterwards arrays[:n_all] = [candidates from the left | own particles | candidates from the right].

    Ordering contract for the later field halos (why the concatenation order is fixed): inside a cell the final
    stable sort keeps [left candidates, own, right candidates].  For the particles of a boundary plane this is the
    same relative order on the owner and on the neighbour that holds them as ghosts -- an immigrant precedes the
    natives on its new owner (it came in the left/right candidate block ... of the side it came from) exactly as it
    does on its old owner (where it is an own particle and the natives are candidates from that side) -- so the
    owner's sorted boundary plane and the neighbour's sorted ghost plane are the same sequence."""
    widths = [1 if a.dim() == 1 else a.shape[1] for a in arrays]

    def pack(lo, hi):
        return torch.cat([a[lo:hi].reshape(hi - lo, w_) for a, w_ in zip(arrays, widths)], 1).contiguous()

    def pieces(rows):
        out, c = [], 0
        for a, w_ in zip(arrays, widths):
            out.append(rows[:, c:c + w_].reshape((rows.shape[0],) + tuple(a.shape[1:])))
            c += w_
        return out

    from_l, from_r = ex.exchange_rows(pack(*to_left), pack(*to_right))
    n_own = own[1] - own[0]
    n_all = from_l.shape[0] + n_own + from_r.shape[0]
    cap = arrays[0].shape[0]
    if n_all > cap:
        raise RuntimeError(f"slab rank {ex.rank}: capacity {cap} exceeded by {n_all} local particles")
    o = 0
    for rows in (from_l, None, from_r):
        if rows is None:
            for a, d in zip(arrays, alt):
                d[o:o + n_own] = a[own[0]:own[1]]
            o += n_own
        else:
            m = rows.shape[0]
            if m:
                for d, pc in zip(alt, pieces(rows)):
                    d[o:o + m] = pc
            o += m
    for a, d in zip(arrays, alt):
        a[:n_all] = d[:n_all]
    return n_all


def plane_ranges(b: tuple, w: int):
    """From the plane offsets (s0, s1, s2, s3, s_{w-1}, s_w, s_{w+1}, s_end) of a sorted local set: the owned range,
    the two outermost owned planes per side (next step's candidates), first / last owned plane, ghost ranges."""
    s0, s1, s2, s3, swm1, sw, sw1, send = b
    own = (s1, sw1)
    to_left = (s1, min(s3, sw1) if w >= 2 else sw1)
    to_right = (max(swm1, s1) if w >= 2 else s1, sw1)
    return {"own": own, "to_left": to_left, "to_right": to_right, "first": (s1, s2 if w >= 2 else sw1),
            "last": (sw if w >= 2 else s1, sw1), "ghost_l": (s0, s1), "ghost_r": (sw1, send)}


_DIAG_NO_HALO = os.environ.get("SPHK_SLAB_DIAG_NOHALO", "0") == "1"


class SlabSystem(SphkOps):
    """One rank of a slab-decomposed SPH system (DFSPH / WCSPH / PBD) over the libsphk C-ABI."""

    HISTORY = {"dfsph": 1, "wcsph": 0, "pbd": 3}      # extra floats per particle that migrate with it

    def __init__(self, scene, rank: int, world: int, device, capacity_factor: float = 1.6, group=None, cut_skew: int = 0,
                 bodies=None, emitters=None, sinks=None, adaptive=None):
        """cut_skew: shifts the interior cuts by that many planes off the balanced position (tests of the re-balancing).
        Kinematic bodies (engine.SphkSystem's `bodies`) are single-GPU only: every rank would have to hold every body.  So are
        open boundaries (engine.SphkSystem's `emitters` / `sinks`): a rank's count is set by the decomposition.  So is CFL-adaptive time
        stepping (engine.SphkSystem's `adaptive`)."""
        if bodies:
            raise ValueError("kinematic bodies are not supported on slab ranks (single-GPU engine.SphkSystem only)")
        if emitters or sinks:
            raise ValueError("emitters and sinks are not supported on slab ranks (single-GPU engine.SphkSystem only)")
        if adaptive:
            raise ValueError("adaptive time stepping is not supported on slab ranks (the speed bound would need a global maximum; "
                             "single-GPU engine.SphkSystem only)")
        self.L = capi.sphk()
        self.p = scene.params
        self.rank, self.world = rank, world
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.current_stream(self.device)
        self.solver = self.p.solver
        self.ex = SlabExchange(rank, world, self.device, group)
        p = self.p
        cx, cy, cz = (int(c) for c in p.cell_size)
        self.plane_cells = cy * cz
        # ---- static partition from the particle CDF along x (host approximation of the hash; exactness is
        # not needed here: a particle one plane off is simply migrated by the first step) --------------------
        device_scene = scene.fluid is None
        n_total = scene.n_fluid
        # strays per rank and step that can be routed (SPHK_SLAB_STRAYS=0: off -- a particle that crosses two planes in a
        # step then stops the run with the ghost-plane mismatch error); world * stray_cap slots are appended to every search
        self.stray_cap = int(os.environ.get("SPHK_SLAB_STRAYS", "2048")) if world > 1 else 0
        self._strays_pending = False
        self._n_scene_fluid = n_total
        if device_scene:
            # SURVEY 8f-4: no host-side particle array.  The CDF comes from the nx lattice columns; the rank generates
            # its own columns on the device, the boundary shell is generated, searched and weighed on the device and the
            # rank's planes are cut out of the sorted set as one contiguous slice.
            (nx, ny, nz), origin = scene.lattice
            col_plane = scene_mod.lattice_column_planes(nx, origin[0], p.cell_length, cx)
            self.cuts = skew_cuts(choose_cuts_weighted(col_plane, ny * nz, cx, world), cut_skew, cx)
            x0, x1 = self.cuts[rank], self.cuts[rank + 1]
            self.x0, self.x1, self.w = x0, x1, x1 - x0
            cols = np.nonzero((col_plane >= x0) & (col_plane < x1))[0]
            j_begin, j_count = (int(cols[0]), int(cols.shape[0])) if cols.shape[0] else (0, 0)
            n_mine = ny * j_count * nz
            cap = int(max(n_mine, n_total / world) * capacity_factor) + 4096 + world * self.stray_cap
            fluid_dev = device_fluid_block(self.L, scene.lattice, self.device, self.stream, j_begin, j_count, capacity=cap)
            bpos, bmass = self._global_boundary_device(scene, x0, x1)
        else:
            plane = np.clip((scene.fluid[:, 0] / np.float32(p.cell_length)).astype(np.int64), 0, cx - 1)
            self.cuts = skew_cuts(choose_cuts(plane, cx, world), cut_skew, cx)
            x0, x1 = self.cuts[rank], self.cuts[rank + 1]
            self.x0, self.x1, self.w = x0, x1, x1 - x0
            mine = scene.fluid[(plane >= x0) & (plane < x1)]
            n_mine = mine.shape[0]
            cap = int(max(n_mine, n_total / world) * capacity_factor) + 4096 + world * self.stray_cap
            # ---- boundary: masses from the GLOBAL boundary set (every rank computes them once), then the subset
            # in this rank's planes [x0-1, x1+1) ---------------------------------------------------------------
            bpos, bmass = self._global_boundary(scene)
            bplane = self._bplane
            sel = (bplane >= x0 - 1) & (bplane < x1 + 1)
            bpos, bmass = bpos[sel], bmass[sel]
            if bpos.shape[0] == 0:                         # keep the C-ABI happy: one far-away massless dummy
                bpos = np.full((1, 3), -1.0e3, np.float32); bmass = np.zeros(1, np.float32)
        self.cap = cap
        # ---- local context ---------------------------------------------------------------------------------
        self.local_cs = (self.w + 2, cy, cz)
        g = SphkGrid()
        g.cell_size[:] = list(self.local_cs)
        g.cell_length = p.cell_length
        g.origin[:] = [x0 - 1, 0, 0]
        self.ncells_local = (self.w + 2) * cy * cz
        if device_scene:
            self.fluid = ParticleSet(fluid_dev, self.device)                      # capacity-sized, first n_mine rows generated
        else:
            self.fluid = ParticleSet(np.zeros((cap, 3), np.float32), self.device)   # capacity-sized arrays
            self.fluid.pos[:n_mine] = torch.from_numpy(np.ascontiguousarray(mine)).to(self.device)
        self.fluid.n = n_mine                                                    # current local count
        self.fluid.mass.fill_(p.m0)                     # SPHSystem.cu:73
        self.boundary = ParticleSet(bpos, self.device)
        self.boundary.mass.copy_(bmass if isinstance(bmass, torch.Tensor) else torch.from_numpy(bmass))
        self.cs_fluid = torch.zeros(self.ncells_local + 1, dtype=torch.int32, device=self.device)
        self.cs_boundary = torch.zeros(self.ncells_local + 1, dtype=torch.int32, device=self.device)
        self.ctx = C.c_void_p()
        # (boundary capacity: the whole shell -- the rank's slice grows and shrinks when the cuts move)
        check(self.L.sphk_create(C.byref(self.ctx), C.c_int(cap), C.c_int(max(self.boundary.n, int(self._bglobal[0].shape[0]))), C.byref(g),
                                 C.c_void_p(self.stream.cuda_stream)), "sphk_create")
        self._alloc_solver_buffers(cap)
        self.use_list = True
        # native exchanges (csrc/sphk_mg.cu): NCCL called directly on the context stream + peer-memory mailboxes for
        # the per-sweep halos.  The torch.distributed path below stays for gloo (CPU tests, ranks sharing one GPU).
        self.mg = None
        # host-free step assembly (no host synchronisation inside a step; SPHK_SLAB_ASYNC=0 selects the synchronous path)
        self.async_assembly = os.environ.get("SPHK_SLAB_ASYNC", "1") == "1"
        self.rebalance_every = int(os.environ.get("SPHK_SLAB_REBALANCE", "50"))   # steps between cut adjustments (0: never)
        self._step_no, self.rebalanced, self.imbalance = -1, 0, 1.0
        self._async_pending = False
        self._step_async = False
        self.time_assembly = False
        self._assembly_events = []
        if world > 1 and not self.ex.stage and dist.get_backend(group) == "nccl" and os.environ.get("SPHK_SLAB_NATIVE", "1") == "1":
            self._init_native(group, cap)
        # interior-first sweeps that overlap the halo exchange: implemented and parity-tested, but measured neutral at
        # N=2 (two extra small launches per sweep cost what the hidden exchange saves), hence opt-in
        self.overlap = os.environ.get("SPHK_SLAB_OVERLAP", "0") == "1"
        self._scene = None
        self._G = (C.c_float * 3)(*[float(x) for x in p.gravity])
        self._space = (C.c_float * 3)(*[float(x) for x in p.space])
        self.n_own, self.n_gl, self.n_gr = n_mine, 0, 0
        self._ranges = None            # plane ranges of the last sorted local set
        # boundary: already in global sorted order -> identity permutation; masses given (not recomputed)
        # (the search's gather packs mass[s] of the sorted slot s into the records: the masses set above)
        self.search_boundary()
        self.comm_s = 0.0
        self.step()                                     # the constructor's implicit step 0 (Q3)

    # ---- construction helpers --------------------------------------------------------------------------
    def _init_native(self, group, cap):
        """sphk_mg communicator: NCCL id from rank 0, mailbox IPC handles all-gathered (torch.distributed is the side
        channel only), transport from SPHK_SLAB_TRANSPORT (1 = peer-memory mailboxes, default; 0 = NCCL halos)."""
        L = self.L
        ident = [None]
        if self.rank == 0:
            buf = (C.c_ubyte * 128)()
            check(L.sphk_mg_unique_id(buf), "sphk_mg_unique_id")
            ident[0] = bytes(buf)
        dist.broadcast_object_list(ident, src=0, group=group)
        transport = int(os.environ.get("SPHK_SLAB_TRANSPORT", "1"))
        # floats per message (3 per plane particle).  Derived from GLOBAL quantities only: every rank must use the same
        # capacity, because a rank computes addresses inside its neighbours' mailboxes from its own layout
        mailbox = 3 * max(262144, int(self._n_scene_fluid / self.world * 1.6) // 4) if transport == 1 else 0
        self.mg = C.c_void_p()
        idbuf = (C.c_ubyte * 128).from_buffer_copy(ident[0])
        check(L.sphk_mg_init(C.byref(self.mg), C.c_int(self.rank), C.c_int(self.world), idbuf,
                             C.c_void_p(self.stream.cuda_stream), C.c_longlong(mailbox)), "sphk_mg_init")
        if transport == 1:
            # wiring can fail on one rank only (no peer access, IPC disabled in the container ...): the ranks agree on the
            # outcome and ALL fall back to NCCL halos together -- mixed transports would wait for each other forever
            ok, why = True, ""
            try:
                hb = (C.c_ubyte * 64)()
                check(L.sphk_mg_ipc_handle(self.mg, hb), "sphk_mg_ipc_handle")
            except RuntimeError as e:
                ok, why, hb = False, str(e), (C.c_ubyte * 64)()
            handles = [None] * self.world
            dist.all_gather_object(handles, (bytes(hb), mailbox, ok), group=group)
            if any(h[1] != mailbox for h in handles):
                raise RuntimeError(f"slab rank {self.rank}: mailbox capacities differ across ranks: {[h[1] for h in handles]}")
            if all(h[2] for h in handles):
                hl = (C.c_ubyte * 64).from_buffer_copy(handles[self.rank - 1][0]) if self.rank > 0 else None
                hr = (C.c_ubyte * 64).from_buffer_copy(handles[self.rank + 1][0]) if self.rank < self.world - 1 else None
                try:
                    check(L.sphk_mg_ipc_connect(self.mg, hl, hr), "sphk_mg_ipc_connect")
                except RuntimeError as e:
                    ok, why = False, str(e)
            else:
                ok = False
            oks = [None] * self.world
            dist.all_gather_object(oks, ok, group=group)   # also: every mailbox is open before the first message
            if not all(oks):
                if self.rank == 0:
                    print(f"[slabs] peer-memory mailboxes unavailable ({why or 'on another rank'}): NCCL halos instead", file=sys.stderr, flush=True)
                transport = 0
        check(L.sphk_mg_set_transport(self.mg, C.c_int(transport)), "sphk_mg_set_transport")
        self.transport = transport
        self._cand_from = None
        self._dev24 = torch.zeros(24, dtype=torch.int32, device=self.device)
        self._pin24 = torch.zeros(24, dtype=torch.int32).pin_memory()
        self._pin_misc = torch.zeros(8, dtype=torch.int32).pin_memory()      # [0] from left, [2] from right, [4] mailbox error word
        self._async_event = torch.cuda.Event()

    def _global_boundary_device(self, scene, x0: int, x1: int):
        """Device-side twin of _global_boundary: the shell is generated (sphk_scene_boundary_shell), searched and weighed
        (SPHSystem.cu:69-71) on this GPU; the sorted set is x-major, so the boundary particles of this rank's planes
        [x0 - 1, x1 + 1) are ONE contiguous slice of it -- cut out device to device (the host reads two offsets)."""
        p = self.p
        g = SphkGrid()
        g.cell_size[:] = [int(c) for c in p.cell_size]
        g.cell_length = p.cell_length
        g.origin[:] = [0, 0, 0]
        b = ParticleSet(device_boundary_shell(self.L, p, self.device, self.stream), self.device)
        nb = b.n
        cs = torch.zeros(p.ncells + 1, dtype=torch.int32, device=self.device)
        ctx = C.c_void_p()
        check(self.L.sphk_create(C.byref(ctx), C.c_int(1), C.c_int(nb), C.byref(g), C.c_void_p(self.stream.cuda_stream)))
        pa = b.abi()
        check(self.L.sphk_neighbor_search(ctx, 1, C.byref(pa), _ptr(cs)))
        check(self.L.sphk_boundary_mass(ctx, C.byref(pa), _ptr(cs), C.c_float(p.rho_boundary), C.c_float(p.radius)))
        pc = int(p.cell_size[1]) * int(p.cell_size[2])
        lo_plane, hi_plane = max(x0 - 1, 0), min(x1 + 1, int(p.cell_size[0]))
        a, e = (int(v) for v in cs[torch.tensor([lo_plane * pc, hi_plane * pc], device=self.device)].cpu().tolist())
        check(self.L.sphk_synchronize(ctx))
        self.L.sphk_destroy(ctx)
        planes = torch.arange(0, int(p.cell_size[0]) + 1, device=self.device) * pc
        self._bglobal = (b.pos, b.mass, cs[planes].cpu().numpy())       # sorted shell + plane offsets: re-sliced when the cuts move
        return self._boundary_slice(x0, x1)

    def _boundary_slice(self, x0: int, x1: int):
        """Boundary particles of the global planes [x0 - 1, x1 + 1) out of the sorted global shell (device tensors)."""
        bpos, bmass, plane_start = self._bglobal
        cx = plane_start.shape[0] - 1
        a, e = int(plane_start[max(x0 - 1, 0)]), int(plane_start[min(x1 + 1, cx)])
        if e <= a:                                      # keep the C-ABI happy: one far-away massless dummy
            return (torch.full((1, 3), -1.0e3, dtype=torch.float32, device=self.device),
                    torch.zeros(1, dtype=torch.float32, device=self.device))
        return bpos[a:e].clone(), bmass[a:e].clone()

    def _global_boundary(self, scene):
        """Sorted global boundary positions + their masses (SPHSystem.cu:69-71) computed on this GPU."""
        p = self.p
        g = SphkGrid()
        g.cell_size[:] = [int(c) for c in p.cell_size]
        g.cell_length = p.cell_length
        g.origin[:] = [0, 0, 0]
        nb = scene.boundary.shape[0]
        b = ParticleSet(scene.boundary, self.device)
        cs = torch.zeros(p.ncells + 1, dtype=torch.int32, device=self.device)
        ctx = C.c_void_p()
        check(self.L.sphk_create(C.byref(ctx), C.c_int(1), C.c_int(nb), C.byref(g), C.c_void_p(self.stream.cuda_stream)))
        pa = b.abi()
        check(self.L.sphk_neighbor_search(ctx, 1, C.byref(pa), _ptr(cs)))
        check(self.L.sphk_boundary_mass(ctx, C.byref(pa), _ptr(cs), C.c_float(p.rho_boundary), C.c_float(p.radius)))
        check(self.L.sphk_synchronize(ctx))
        pos, mass = b.pos.cpu().numpy(), b.mass.cpu().numpy()
        csh = cs.cpu().numpy()
        # plane of each SORTED boundary particle from the cell ranges
        plane_start = csh[np.arange(0, p.cell_size[0] + 1) * (int(p.cell_size[1]) * int(p.cell_size[2]))]
        self._bplane = np.searchsorted(plane_start, np.arange(nb), side="right") - 1
        self._bglobal = (torch.from_numpy(pos).to(self.device), torch.from_numpy(mass).to(self.device), plane_start)
        self.L.sphk_destroy(ctx)
        return pos, mass

    # ---- step ---------------------------------------------------------------------------------------------
    def _carried(self):
        """Per-particle arrays that migrate with a particle."""
        arrs = [self.fluid.pos, self.fluid.vel]
        if self.solver == "dfsph":
            arrs.append(self.warm)
        elif self.solver == "pbd":
            arrs.append(self.pos_last)
        return arrs

    def _array_args(self, arrays):
        k = len(arrays)
        return C.c_int(k), (C.c_void_p * k)(*[a.data_ptr() for a in arrays]), (C.c_int * k)(*_widths(arrays))

    def _collect_strays(self):
        """sphk_strays_collect over the owned range of the current sorted set (see "strays" at the top of the module)."""
        self._refresh_ranges()
        arrays = self._carried()
        if not hasattr(self, "_stray_block"):
            nf = stray_block_floats(self.stray_cap, _widths(arrays))
            self._stray_block = torch.zeros(nf, dtype=torch.float32, device=self.device)
            self._stray_gathered = torch.zeros(self.world * nf, dtype=torch.float32, device=self.device)
        a, b = self._ranges["own"]
        k, ptrs, widths = self._array_args(arrays)
        check(self.L.sphk_strays_collect(self.ctx, _ptr(self.cs_fluid), C.c_int(a), C.c_int(b - a), k, ptrs, widths,
                                         _ptr(self._stray_block), C.c_int(self.stray_cap)), "sphk_strays_collect")
        self._strays_pending = True

    def _route_strays(self, arrays, n_all: int) -> int:
        """All-gather of the collected blocks + append at slot n_all of `arrays` (the set being assembled for the search).
        Returns the new slot count."""
        if not self._strays_pending:
            return n_all
        self._strays_pending = False
        extra = self.world * self.stray_cap
        if n_all + extra > self.cap:
            raise RuntimeError(f"slab rank {self.rank}: capacity {self.cap} exceeded by {n_all} local particles + {extra} stray slots")
        k, ptrs, widths = self._array_args(arrays)
        if self.mg is not None:
            check(self.L.sphk_mg_strays_route(self.mg, self.ctx, _ptr(self._stray_block), _ptr(self._stray_gathered), C.c_int(self.stray_cap),
                                              k, ptrs, widths, C.c_int(n_all)), "sphk_mg_strays_route")
        else:
            self._stray_gathered.copy_(self.ex.all_gather(self._stray_block))
            check(self.L.sphk_strays_append(self.ctx, _ptr(self._stray_gathered), C.c_int(self.world), C.c_int(self.stray_cap), k, ptrs, widths,
                                            C.c_int(n_all)), "sphk_strays_append")
        return n_all + extra

    def stray_counts(self):
        """Strays each rank collected in the last step that had any routing (synchronises; introspection)."""
        if not hasattr(self, "_stray_gathered"):
            return [0] * self.world
        out = (C.c_int * self.world)()
        k, _, widths = self._array_args(self._carried())
        check(self.L.sphk_strays_counts(self.ctx, _ptr(self._stray_gathered), C.c_int(self.world), C.c_int(self.stray_cap), k, widths, out))
        return list(out)

    def _search_all(self, n):
        """The C-ABI neighbour search over slots [0, n).  The history array (DFSPH warm stiffness, PBD last positions)
        is NOT permuted here: the solver sequence does that itself with the same permutation (DFSPHSolver.cu:170-171,
        PBDSolver.cu:84-85), exactly as on one GPU."""
        self.fluid.n = n
        self._scene = None
        self.search_fluid()

    def _bounds(self):
        if not hasattr(self, "_bounds_idx"):
            pc, w = self.plane_cells, self.w
            self._bounds_idx = torch.tensor([0, pc, 2 * pc, 3 * pc, max(w - 1, 0) * pc, w * pc, (w + 1) * pc, (w + 2) * pc],
                                            device=self.device)
        return tuple(self.cs_fluid[self._bounds_idx].cpu().tolist())

    def _exchange_ints(self, to_left, to_right):
        k = len(to_left)
        tl, tr = (C.c_int * k)(*to_left), (C.c_int * k)(*to_right)
        fl, fr = (C.c_int * k)(), (C.c_int * k)()
        check(self.L.sphk_mg_exchange_ints(self.mg, tl, tr, fl, fr, C.c_int(k)), "sphk_mg_exchange_ints")
        return list(fl), list(fr)

    def _swap_carried(self):
        """The assembled set was received into the scratch twins: make them the live arrays (no copy back)."""
        self.fluid.pos, self._alt[0] = self._alt[0], self.fluid.pos
        self.fluid.vel, self._alt[1] = self._alt[1], self.fluid.vel
        if self.solver == "dfsph":
            self.warm, self._alt[2] = self._alt[2], self.warm
        elif self.solver == "pbd":
            self.pos_last, self._alt[2] = self._alt[2], self.pos_last
        self._scene = None

    def _begin_step_native(self):
        """begin_step over csrc/sphk_mg.cu: candidates travel array by array in ONE NCCL group straight into their slots
        of the assembled set (no packing, no copy back); the receive counts were agreed in the previous step, so the only
        host synchronisation left is reading the plane offsets after the search."""
        t0 = time.perf_counter()
        L = self.L
        ev = None
        self._refresh_ranges()
        self._step_async = False
        if self.time_assembly:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        arrays = self._carried()
        if not hasattr(self, "_alt"):
            self._alt = [torch.empty_like(a) for a in arrays]
        if self._ranges is None:                         # very first step: as in begin_step below
            self._search_all(self.n_own)
            b = self._bounds()
            if b[7] != self.n_own:
                raise RuntimeError(f"slab rank {self.rank}: initial partition left particles outside the local grid")
            r = plane_ranges(b, self.w)
            r["own"] = (b[0], b[7])
            r["to_left"] = (b[0], r["to_left"][1])
            r["to_right"] = (r["to_right"][0], b[7])
            self._ranges = r
            fl, fr = self._exchange_ints([r["to_left"][1] - r["to_left"][0]], [r["to_right"][1] - r["to_right"][0]])
            self._cand_from = (fl[0], fr[0])
        r = self._ranges
        nl, nr = self._cand_from
        if self.ex.left is None:
            nl = 0
        if self.ex.right is None:
            nr = 0
        own0, own1 = r["own"]
        n_own = own1 - own0
        n_all = nl + n_own + nr
        if n_all > self.cap:
            raise RuntimeError(f"slab rank {self.rank}: capacity {self.cap} exceeded by {n_all} local particles")
        k = len(arrays)
        widths = (C.c_int * k)(*[1 if a.dim() == 1 else a.shape[1] for a in arrays])
        src = (C.c_void_p * k)(*[a.data_ptr() for a in arrays])
        dst = (C.c_void_p * k)(*[a.data_ptr() for a in self._alt])
        i2 = C.c_int * 2
        check(L.sphk_mg_exchange_slices(self.mg, C.c_int(k), src, dst, widths,
                                        i2(r["to_left"][0], r["to_left"][1] - r["to_left"][0]),
                                        i2(r["to_right"][0], r["to_right"][1] - r["to_right"][0]),
                                        i2(0, nl), i2(nl + n_own, nr)), "sphk_mg_exchange_slices")
        for a, d in zip(arrays, self._alt):
            wd = 1 if a.dim() == 1 else a.shape[1]
            check(L.sphk_copy(self.ctx, C.c_void_p(d.data_ptr() + 4 * wd * nl), C.c_void_p(a.data_ptr() + 4 * wd * own0),
                              C.c_int(n_own * wd)), "sphk_copy")
        n_all = self._route_strays(self._alt, n_all)
        self._swap_carried()
        self._search_all(n_all)
        b = self._bounds()
        self._ranges = r = plane_ranges(b, self.w)
        self.n_gl = r["ghost_l"][1] - r["ghost_l"][0]
        self.n_own = r["own"][1] - r["own"][0]
        self.n_gr = r["ghost_r"][1] - r["ghost_r"][0]
        self.first_plane, self.last_plane = r["first"], r["last"]
        self.ghost_l, self.ghost_r = r["ghost_l"], r["ghost_r"]
        # one small exchange: (a) the ordering contract -- my ghost planes must be exactly the neighbours' boundary
        # planes -- checked BEFORE any halo is posted (a mismatch would otherwise stall the exchange); (b) how many
        # candidates each neighbour will send next step
        n_first, n_last = self.first_plane[1] - self.first_plane[0], self.last_plane[1] - self.last_plane[0]
        fl, fr = self._exchange_ints([n_first, r["to_left"][1] - r["to_left"][0]], [n_last, r["to_right"][1] - r["to_right"][0]])
        if (self.ex.left is not None and fl[0] != self.n_gl) or (self.ex.right is not None and fr[0] != self.n_gr):
            raise RuntimeError(f"slab rank {self.rank}: ghost planes {self.n_gl}/{self.n_gr} do not match the neighbours' "
                               f"boundary planes {fl[0]}/{fr[0]} (a particle moved more than one plane in a step?)")
        self._cand_from = (fl[1], fr[1])
        err = C.c_int(0)
        check(L.sphk_mg_check(self.mg, C.byref(err)), "sphk_mg_check")
        if err.value:
            raise RuntimeError(f"slab rank {self.rank}: halo mailbox error bits {err.value:#x} (see sphk_mg_check)")
        self._halo_ranges = (C.c_int * 8)(self.first_plane[0], n_first, self.last_plane[0], n_last,
                                          self.ghost_l[0], self.n_gl, self.ghost_r[0], self.n_gr)
        check(L.sphk_set_active_range(self.ctx, C.c_int(r["own"][0]), C.c_int(self.n_own)))
        if self.use_list:
            self.set_use_list(True, 150 if self.solver == "pbd" else 0)
            self.build_neighbor_list()
        if ev is not None:
            ev[1].record()
            self._assembly_events.append(ev)
        self.comm_s += time.perf_counter() - t0

    def assembly_ms(self) -> float:
        """Device time (CUDA events) of the recorded begin_step phases: candidate exchange + search + plane offsets +
        count exchange + list build, host round trips included.  Synchronises."""
        torch.cuda.synchronize(self.device)
        ms = sum(a.elapsed_time(b) for a, b in self._assembly_events)
        n = max(len(self._assembly_events), 1)
        self._assembly_events = []
        return ms / n

    def _halo(self, what: int, t: torch.Tensor):
        if _DIAG_NO_HALO:                # timing diagnostic only (results are WRONG): what the halos cost a step
            return
        if self._step_async:             # this step's ranges live on the device
            check(self.L.sphk_mg_halo_device(self.mg, self.ctx, self._s(), C.c_int(what), _ptr(t), C.c_int(1 if t.dim() == 1 else t.shape[1]),
                                             C.c_void_p(self._dev24.data_ptr() + 4 * 8), C.c_int(self.cap)), "sphk_mg_halo_device")
            return
        check(self.L.sphk_mg_halo(self.mg, self.ctx, self._s(), C.c_int(what), _ptr(t), C.c_int(1 if t.dim() == 1 else t.shape[1]),
                                  self._halo_ranges), "sphk_mg_halo")

    # ---- host-free step assembly -----------------------------------------------------------------------------------------
    def _refresh_ranges(self):
        """Plane ranges / neighbour counts of the CURRENT sorted set, produced on the device during the last begin_step
        and copied to pinned host memory: waits for that copy (long finished unless called right after begin_step)."""
        if not getattr(self, "_async_pending", False):
            return
        self._async_event.synchronize()
        self._async_pending = False
        pin = self._pin24.tolist()
        err = int(self._pin_misc[4])
        if err:
            raise RuntimeError(f"slab rank {self.rank}: halo mailbox error bits {err:#x} (see sphk_mg_check)")
        self._ranges = r = plane_ranges(tuple(pin[0:8]), self.w)
        self.n_gl = r["ghost_l"][1] - r["ghost_l"][0]
        self.n_own = r["own"][1] - r["own"][0]
        self.n_gr = r["ghost_r"][1] - r["ghost_r"][0]
        self.first_plane, self.last_plane = r["first"], r["last"]
        self.ghost_l, self.ghost_r = r["ghost_l"], r["ghost_r"]
        self._cand_from = (int(self._pin_misc[0]), int(self._pin_misc[2]))

    def _begin_step_async(self):
        """begin_step without a host synchronisation.  The host only needs LAST step's plane ranges (to slice the
        candidates and size this step's search) -- they were computed on the device right after last step's search and
        arrived in pinned memory while the solver kernels of that step were running.  Everything THIS step derives from
        its own search (owned range, halo ranges, next candidates, the neighbours' counts) stays on the device:
        sphk_mg_plane_ranges -> sphk_set_active_range_device / sphk_mg_halo_device / sphk_mg_exchange_ints_async."""
        t0 = time.perf_counter()
        L = self.L
        ev = None
        if self.time_assembly:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        self._refresh_ranges()
        arrays = self._carried()
        r = self._ranges
        nl, nr = self._cand_from
        if self.ex.left is None:
            nl = 0
        if self.ex.right is None:
            nr = 0
        own0, own1 = r["own"]
        n_own = own1 - own0
        n_all = nl + n_own + nr
        if n_all > self.cap:
            raise RuntimeError(f"slab rank {self.rank}: capacity {self.cap} exceeded by {n_all} local particles")
        k = len(arrays)
        widths = (C.c_int * k)(*[1 if a.dim() == 1 else a.shape[1] for a in arrays])
        src = (C.c_void_p * k)(*[a.data_ptr() for a in arrays])
        dst = (C.c_void_p * k)(*[a.data_ptr() for a in self._alt])
        i2 = C.c_int * 2
        check(L.sphk_mg_exchange_slices(self.mg, C.c_int(k), src, dst, widths,
                                        i2(r["to_left"][0], r["to_left"][1] - r["to_left"][0]),
                                        i2(r["to_right"][0], r["to_right"][1] - r["to_right"][0]),
                                        i2(0, nl), i2(nl + n_own, nr)), "sphk_mg_exchange_slices")
        for a, d in zip(arrays, self._alt):
            wd = 1 if a.dim() == 1 else a.shape[1]
            check(L.sphk_copy(self.ctx, C.c_void_p(d.data_ptr() + 4 * wd * nl), C.c_void_p(a.data_ptr() + 4 * wd * own0),
                              C.c_int(n_own * wd)), "sphk_copy")
        n_all = self._route_strays(self._alt, n_all)
        self._swap_carried()
        self._search_all(n_all)
        d24 = self._dev24.data_ptr()
        check(L.sphk_mg_plane_ranges(self.mg, _ptr(self.cs_fluid), C.c_int(self.plane_cells), C.c_int(self.w), C.c_void_p(d24),
                                     C.c_void_p(self._pin24.data_ptr())), "sphk_mg_plane_ranges")
        pm = self._pin_misc.data_ptr()
        check(L.sphk_mg_exchange_ints_async(self.mg, C.c_void_p(d24 + 4 * 22), C.c_void_p(d24 + 4 * 23), C.c_int(1),
                                            C.c_void_p(pm), C.c_void_p(pm + 8)), "sphk_mg_exchange_ints_async")
        check(L.sphk_mg_check_async(self.mg, C.c_void_p(pm + 16)), "sphk_mg_check_async")
        self._async_event.record()
        self._async_pending = True
        self._step_async = True
        check(L.sphk_set_active_range_device(self.ctx, C.c_void_p(d24 + 4 * 16)), "sphk_set_active_range_device")
        if self.use_list:
            self.set_use_list(True, 150 if self.solver == "pbd" else 0)
            self.build_neighbor_list()
        if ev is not None:
            ev[1].record()
            self._assembly_events.append(ev)
        self.comm_s += time.perf_counter() - t0

    def begin_step(self):
        if self.mg is not None and self.async_assembly and self._ranges is not None and getattr(self, "transport", 0) == 1:
            return self._begin_step_async()
        if self.mg is not None:
            return self._begin_step_native()
        t0 = time.perf_counter()
        arrays = self._carried()
        if not hasattr(self, "_alt"):
            self._alt = [torch.empty_like(a) for a in arrays]
        if self._ranges is None:                         # very first step: sort the initial set once
            self._search_all(self.n_own)                 # (history arrays are still all-zero: nothing to permute)
            b = self._bounds()
            if b[7] != self.n_own:
                raise RuntimeError(f"slab rank {self.rank}: initial partition left particles outside the local grid")
            r = plane_ranges(b, self.w)
            # the host-side initial partition may be one plane off for a few particles (it does not use the device
            # hash): treat everything local as "own" and include the ghost planes in the candidates once
            r["own"] = (b[0], b[7])
            r["to_left"] = (b[0], r["to_left"][1])
            r["to_right"] = (r["to_right"][0], b[7])
            self._ranges = r
        r = self._ranges
        n_all = exchange_candidates(self.ex, arrays, self._alt, r["own"], r["to_left"], r["to_right"])
        n_all = self._route_strays(arrays, n_all)
        self._search_all(n_all)
        b = self._bounds()
        self._ranges = r = plane_ranges(b, self.w)
        self.n_gl = r["ghost_l"][1] - r["ghost_l"][0]
        self.n_own = r["own"][1] - r["own"][0]
        self.n_gr = r["ghost_r"][1] - r["ghost_r"][0]
        check(self.L.sphk_set_active_range(self.ctx, C.c_int(r["own"][0]), C.c_int(self.n_own)))
        self.first_plane, self.last_plane = r["first"], r["last"]
        self.ghost_l, self.ghost_r = r["ghost_l"], r["ghost_r"]
        if os.environ.get("SPHK_SLAB_DEBUG"):
            print(f"[slab {self.rank}] bounds {b} first {self.first_plane} last {self.last_plane} ghosts {self.ghost_l} {self.ghost_r} "
                  f"to_left {r['to_left']} to_right {r['to_right']} n_all {n_all}", flush=True)
        if self.use_list:
            self.set_use_list(True, 150 if self.solver == "pbd" else 0)
            self.build_neighbor_list()
        self.comm_s += time.perf_counter() - t0

    # field syncs ------------------------------------------------------------------------------------------------
    def _sync(self, t: torch.Tensor):
        fl = t[self.first_plane[0]:self.first_plane[1]]
        ll = t[self.last_plane[0]:self.last_plane[1]]
        self.ex.exchange(fl, ll, t[self.ghost_l[0]:self.ghost_l[1]], t[self.ghost_r[0]:self.ghost_r[1]])

    def _push(self, what: int, arr):
        for b, e in (self.ghost_l, self.ghost_r):
            if e > b:
                check(self.L.sphk_push_range(self.ctx, self._s(), C.c_int(what), _ptr(arr), C.c_int(b), C.c_int(e - b)))

    # ---- overlapped sweep + halo: boundary planes first, exchange while the interior is being computed -----------
    def _set_active(self, b, e):
        check(self.L.sphk_set_active_range(self.ctx, C.c_int(b), C.c_int(max(e - b, 0))))

    def _run(self, op, sync=None, tensor=None, split=True):
        if sync is None or not split or not self.overlap or self.ex.stage or self.mg is not None:
            return super()._run(op, sync, tensor)
        (f0, f1), (l0, l1) = self.first_plane, self.last_plane
        own0, own1 = self._ranges["own"]
        if l0 < f1:                                   # one- or two-plane slab: no interior to overlap with
            return super()._run(op, sync, tensor)
        self._set_active(f0, f1); op()
        self._set_active(l0, l1); op()
        t = self.fluid.vel if sync == "vel" else tensor
        works = self._sync_start(t)
        self._set_active(f1, l0); op()                # interior: no ghost neighbours, runs while the halo is in flight
        for w in works:
            w.wait()
        if sync == "vel":
            self._push(1, None)
        elif sync == "scalar":
            self._push(2, tensor)
        self._set_active(own0, own1)

    def _sync_start(self, t):
        ex = self.ex
        ops = []
        fl = t[self.first_plane[0]:self.first_plane[1]]
        ll = t[self.last_plane[0]:self.last_plane[1]]
        gl, gr = t[self.ghost_l[0]:self.ghost_l[1]], t[self.ghost_r[0]:self.ghost_r[1]]
        if ex.left is not None:
            if fl.numel(): ops.append(dist.P2POp(dist.isend, fl, ex.left, ex.group)); ex.bytes_sent += fl.numel() * 4; ex.messages += 1
            if gl.numel(): ops.append(dist.P2POp(dist.irecv, gl, ex.left, ex.group))
        if ex.right is not None:
            if ll.numel(): ops.append(dist.P2POp(dist.isend, ll, ex.right, ex.group)); ex.bytes_sent += ll.numel() * 4; ex.messages += 1
            if gr.numel(): ops.append(dist.P2POp(dist.irecv, gr, ex.right, ex.group))
        return dist.batch_isend_irecv(ops) if ops else []

    def sync_vel(self):
        if self.mg is not None:
            return self._halo(1, self.fluid.vel)
        self._sync(self.fluid.vel)
        self._push(1, None)

    def sync_scalar(self, t):
        if self.mg is not None:
            return self._halo(2, t)
        self._sync(t)
        self._push(2, t)

    def sync_array(self, t):
        if self.mg is not None:
            return self._halo(0, t)
        self._sync(t)

    def sync_positions(self):
        """PBD moves positions inside a step (Q7): the ghosts follow their owners after every projection."""
        if self.mg is not None:
            return self._halo(4, self.fluid.pos)
        self._sync(self.fluid.pos)
        self._push(4, None)

    def owned(self, t):
        self._refresh_ranges()
        return t[self._ranges["own"][0]:self._ranges["own"][1]]

    def n_total(self) -> int:
        if not hasattr(self, "_n_total"):
            self._n_total = self.n_global()
        return self._n_total

    def reduce_sum(self, x: float) -> float:
        if self.mg is not None:
            v = C.c_double(x)
            check(self.L.sphk_mg_allreduce_sum(self.mg, C.byref(v)), "sphk_mg_allreduce_sum")
            return float(v.value)
        t = torch.tensor([x], dtype=torch.float64, device=self.device)
        dist.all_reduce(t, group=self.ex.group)
        return float(t.item())

    # ---- load re-balancing (SURVEY 8e: "re-balance every K steps") ------------------------------------------------------------
    def rebalance(self) -> bool:
        """Moves every interior cut by at most ONE plane towards the position that balances the current particle counts
        (a dam-break sloshes: the block that starts in one corner spreads over the whole box).  No particle data moves
        here: a cut that shifts by one plane only changes which of the planes a rank already exchanges as candidates
        count as owned -- the next step's sort does the rest -- provided the candidates cover THREE planes per side for
        that one step (the moved cut uses up the one-plane margin the usual two planes leave for particle motion).
        Collective; synchronises (it reads w + 1 cell offsets and agrees on counts), so it runs every K steps only."""
        if self.world == 1 or self._ranges is None:
            return False
        self._refresh_ranges()
        pc, w = self.plane_cells, self.w
        offs = self.cs_fluid[torch.arange(1, w + 2, device=self.device) * pc].cpu().numpy().astype(np.int64)   # planes 1 .. w+1
        mine = (self.x0, np.diff(offs).tolist())
        everybody = [None] * self.world
        dist.all_gather_object(everybody, mine, group=self.ex.group)
        cx = int(self.p.cell_size[0])
        counts = np.zeros(cx, np.int64)
        for x0_, c in everybody:
            counts[x0_:x0_ + len(c)] = c
        ideal = _cuts_from_counts(counts, cx, self.world)
        new = list(self.cuts)
        for g in range(1, self.world):
            new[g] = self.cuts[g] + int(np.sign(ideal[g] - self.cuts[g]))
            new[g] = min(max(new[g], new[g - 1] + 1), cx - (self.world - g))
        self.imbalance = float(max(sum(c) for _, c in everybody) * self.world / max(int(counts.sum()), 1))
        if new == list(self.cuts):
            return False
        # candidates of the next exchange: three planes per side (offsets of the CURRENT sorted set)
        s1, sw1 = int(offs[0]), int(offs[w])
        s4 = int(offs[min(3, w)])
        swm2 = int(offs[max(w - 3, 0)])
        r = self._ranges
        r["to_left"], r["to_right"] = (s1, min(s4, sw1)), (max(swm2, s1), sw1)
        if self.mg is not None:
            fl, fr = self._exchange_ints([r["to_left"][1] - r["to_left"][0]], [r["to_right"][1] - r["to_right"][0]])
            self._cand_from = (fl[0], fr[0])
        # the new local grid
        self.cuts = new
        self.x0, self.x1 = new[self.rank], new[self.rank + 1]
        self.w = self.x1 - self.x0
        cy, cz = int(self.p.cell_size[1]), int(self.p.cell_size[2])
        self.local_cs = (self.w + 2, cy, cz)
        g = SphkGrid()
        g.cell_size[:] = list(self.local_cs)
        g.cell_length = self.p.cell_length
        g.origin[:] = [self.x0 - 1, 0, 0]
        check(self.L.sphk_set_grid(self.ctx, C.byref(g)), "sphk_set_grid")
        self.ncells_local = (self.w + 2) * cy * cz
        self.cs_fluid = torch.zeros(self.ncells_local + 1, dtype=torch.int32, device=self.device)
        self.cs_boundary = torch.zeros(self.ncells_local + 1, dtype=torch.int32, device=self.device)
        bpos, bmass = self._boundary_slice(self.x0, self.x1)
        self.boundary = ParticleSet(bpos, self.device)
        self.boundary.mass.copy_(bmass)
        self._scene = None
        if hasattr(self, "_bounds_idx"):
            del self._bounds_idx
        self.search_boundary()                          # (masses are given: the search only sorts and packs them)
        self._step_async = False
        self.rebalanced += 1
        return True

    # implicit viscosity needs a global dot product per CG iteration and a halo of the direction before each product
    @property
    def implicit_nu(self):
        return 0.0

    @implicit_nu.setter
    def implicit_nu(self, nu):
        if nu != 0.0:
            raise ValueError("implicit viscosity is not supported on slab ranks (single-GPU engine.SphkSystem only)")

    # non-Newtonian viscosity: the same solve, and a shear sweep that would need the ghosts' velocity gradients
    @property
    def rheology(self):
        return None

    @rheology.setter
    def rheology(self, spec):
        if spec is not None:
            raise ValueError("non-Newtonian viscosity is not supported on slab ranks (single-GPU engine.SphkSystem only)")

    # adhesion: the boundary walk and the body reaction are single-context only
    @property
    def adhesion(self):
        return None

    @adhesion.setter
    def adhesion(self, spec):
        if spec is not None:
            raise ValueError("adhesion is not supported on slab ranks (single-GPU engine.SphkSystem only)")

    # probes and gauges: a probe near a cut would miss the other rank's fluid
    def set_probes(self, points=(), gauges=(), threshold=0.5, capacity=1024):
        raise ValueError("probes and gauges are not supported on slab ranks (single-GPU engine.SphkSystem only)")

    # heat transfer: ghosts and strays would need their temperatures carried as a second array
    @property
    def thermal(self):
        return None

    @thermal.setter
    def thermal(self, spec):
        if spec is not None:
            raise ValueError("heat transfer is not supported on slab ranks (single-GPU engine.SphkSystem only)")

    def step(self):
        self._step_no += 1
        if self.stray_cap and self._ranges is not None:
            self._collect_strays()                      # (before a re-balance moves the window the sorted set refers to)
        if self.rebalance_every > 0 and self._step_no % self.rebalance_every == 0:
            self.rebalance()
        self.begin_step()
        self._step_solver()

    def n_global(self):
        self._refresh_ranges()
        return int(self.reduce_sum(float(self.n_own)))

    def comm_stats(self):
        """(bytes sent, messages sent) by this rank."""
        if self.mg is not None:
            out = (C.c_longlong * 2)()
            check(self.L.sphk_mg_stats(self.mg, out))
            return int(out[0]), int(out[1])
        return self.ex.bytes_sent, self.ex.messages

    def close(self):
        if getattr(self, "mg", None) is not None and self.ctx:
            self.L.sphk_synchronize(self.ctx)
            self.L.sphk_mg_destroy(self.mg)
            self.mg = None
        super().close()

    def owned_state(self) -> dict:
        """Owned particles of this rank (host arrays)."""
        self.synchronize()
        self._refresh_ranges()
        a, b = self._ranges["own"]
        g = lambda t: t[a:b].detach().cpu().numpy()  # noqa: E731
        return {"pos": g(self.fluid.pos), "vel": g(self.fluid.vel), "density": g(self.fluid.density)}


def gather_state(sys_: SlabSystem) -> dict | None:
    """All ranks' owned particles on rank 0, in a canonical order (lexicographic by position)."""
    st = sys_.owned_state()
    objs = [None] * sys_.world
    dist.all_gather_object(objs, st, group=sys_.ex.group)
    if sys_.rank != 0:
        return None
    out = {k: np.concatenate([o[k] for o in objs], 0) for k in ("pos", "vel", "density")}
    order = np.lexsort((out["pos"][:, 2], out["pos"][:, 1], out["pos"][:, 0]))
    return {k: v[order] for k, v in out.items()}


def lattice_keys(pos: np.ndarray, origin, spacing: float) -> np.ndarray:
    """Identity of a dam-break particle a few steps after the start: the index of the lattice site it started from
    (displacements are << spacing / 2 during the first steps), as one int64 per particle."""
    q = np.rint((pos.astype(np.float64) - np.asarray(origin, np.float64)) / float(spacing)).astype(np.int64)
    q -= q.min(0)
    ext = q.max(0) + 1
    return (q[:, 0] * ext[1] + q[:, 1]) * ext[2] + q[:, 2]


def parity_check(sys_: "SlabSystem", scene, steps: int = 2) -> dict | None:
    """Multi-rank result against a single-GPU run of the SAME scene (rank 0's GPU), `steps` steps after the
    constructor's step 0: every rank's owned particles are gathered on rank 0, matched to the single-GPU particles by
    their lattice site, and compared -- <= 1e-5 scale-relative on positions and densities (north_star), velocities
    reported.  Returns the verdict on rank 0 (None elsewhere); raises on a mismatch so that a wrong multi-GPU run can
    never produce a bench line."""
    from . import engine, scene as scene_mod
    for _ in range(steps):
        sys_.step()
    st = sys_.owned_state()
    gathered = [None] * sys_.world if sys_.rank == 0 else None
    dist.gather_object(st, gathered, dst=0, group=sys_.ex.group)
    verdict = [None]
    if sys_.rank == 0:
        multi = {k: np.concatenate([g[k] for g in gathered], 0) for k in ("pos", "vel", "density")}
        ref = engine.SphkSystem(scene, device=sys_.device)
        for _ in range(steps):
            ref.step()
        one = ref.state()
        ref.close()
        del ref
        torch.cuda.empty_cache()
        n = scene.n_fluid
        ok_count = multi["pos"].shape[0] == n
        origin = scene.fluid.min(0) if scene.fluid is not None else np.asarray(scene.lattice[1], np.float32)
        spacing = float(scene_mod.SPACING)
        km = lattice_keys(multi["pos"], origin, spacing) if ok_count else None
        ko = lattice_keys(one["pos"], origin, spacing)
        unique = ok_count and np.unique(km).shape[0] == n and np.unique(ko).shape[0] == n
        errs = {}
        if unique:
            om, oo = np.argsort(km), np.argsort(ko)
            unique = bool(np.array_equal(km[om], ko[oo]))
            if unique:
                for f in ("pos", "density", "vel"):
                    a, b = multi[f][om].astype(np.float64), one[f][oo].astype(np.float64)
                    errs[f] = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
        good = bool(unique and errs["pos"] <= 1e-5 and errs["density"] <= 1e-5)
        verdict[0] = {"parity_checked": True, "parity_ok": good, "steps_after_constructor": steps, "particles_compared": int(n),
                      "against": "single-GPU run of the same scene on rank 0 (engine.SphkSystem), particles matched by lattice site",
                      "max_rel_err": errs, "all_particles_present_once": bool(unique)}
    dist.broadcast_object_list(verdict, src=0, group=sys_.ex.group)
    if not verdict[0]["parity_ok"]:
        raise RuntimeError(f"multi-GPU parity check failed: {verdict[0]}")
    return verdict[0] if sys_.rank == 0 else None


# ----------------------------------------------------------------------------------------------------------------
def bench_main(args, pkg) -> dict | None:
    """bench.py --gpus N (N > 1): one rank per GPU under torchrun; weak scaling, 2M fluid particles per GPU."""
    import bench as B
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    if world != args.gpus:
        if rank == 0:
            print(f'{{"error": "launch with torchrun --nproc-per-node {args.gpus} (WORLD_SIZE={world})"}}')
        return None
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    solver = args.workload
    strong = getattr(args, "scaling", "weak") == "strong"
    scene_name = args.scene or ("2m" if strong else B.SCENE_OF_N[world])
    sc = pkg.scene.benchmark_scene(scene_name, solver, device_init=os.environ.get("SPHK_BENCH_DEVICE_SCENE", "1") == "1")
    n = sc.n_fluid
    # a rank that dies must take the job down at once (its neighbours would wait for it inside a collective), and a job
    # that stops making progress must not sit on the GPUs: bounded by a watchdog
    import threading
    limit = float(os.environ.get("SPHK_BENCH_WATCHDOG_S", "420"))
    dog = threading.Timer(limit, lambda: (print(f"[bench] rank {rank}: no result after {limit:.0f} s, aborting", file=sys.stderr, flush=True), os._exit(3)))
    dog.daemon = True
    dog.start()
    try:
        out = _bench_body(args, pkg, B, sc, n, rank, world, local, solver, scene_name)
        if out is not None and strong:
            out["scaling"] = "strong"
        return out
    except BaseException:
        import traceback
        traceback.print_exc()
        sys.stderr.flush(); sys.stdout.flush()
        os._exit(1)
    finally:
        dog.cancel()


def _bench_body(args, pkg, B, sc, n, rank, world, local, solver, scene_name):
    s = SlabSystem(sc, rank, world, torch.device("cuda", local))
    # the result must be RIGHT before it is timed: two steps against a single-GPU run of the same scene (<= 1e-5)
    parity = parity_check(s, sc, steps=2) if os.environ.get("SPHK_BENCH_PARITY", "1") == "1" else None
    for _ in range(args.warmup):
        s.step()
    sampler = B.ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = s.launch_count()
    s.comm_s = 0.0
    s.time_assembly = s.mg is not None
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        s.step()
    e1.record()
    dist.barrier()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=s.device)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)              # max over ranks
    launches = torch.tensor([s.launch_count() - launches0], dtype=torch.float64, device=s.device)
    dist.all_reduce(launches)
    s._refresh_ranges()
    own = torch.tensor([float(s.n_own), float(s.n_own)], dtype=torch.float64, device=s.device)
    mx = own.clone()
    dist.all_reduce(own)
    dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    clocks = sampler.stop() if rank == 0 else None
    # ---- e2e: every step takes this rank's owned particles from pinned HOST buffers and returns them there ------------
    # (pos + vel in, pos + vel + density out; copies on the compute stream, inside the timed region)
    e2e = None
    hpos = hvel = hden = None
    try:                                                   # the only rank-specific failure: pinned host memory
        cap = s.cap
        hpos = torch.empty((cap, 3), dtype=torch.float32, pin_memory=True)
        hvel = torch.empty((cap, 3), dtype=torch.float32, pin_memory=True)
        hden = torch.empty(cap, dtype=torch.float32, pin_memory=True)
    except Exception as exc:
        print(f"[bench] rank {rank}: no pinned buffers for the e2e leg: {exc}", file=sys.stderr, flush=True)
        hpos = None
    agree = torch.tensor([0.0 if hpos is None else 1.0], dtype=torch.float64, device=s.device)
    dist.all_reduce(agree, op=dist.ReduceOp.MIN)           # all ranks run the leg, or none (a lone rank would wait for ever)
    try:
        if agree.item() < 1.0:
            raise RuntimeError("skipped: a rank could not allocate its pinned buffers")

        def down():
            s._refresh_ranges()
            a, b = s._ranges["own"]
            hpos[:b - a].copy_(s.fluid.pos[a:b], non_blocking=True)
            hvel[:b - a].copy_(s.fluid.vel[a:b], non_blocking=True)
            hden[:b - a].copy_(s.fluid.density[a:b], non_blocking=True)
            return 28 * (b - a)

        def up():
            s._refresh_ranges()
            a, b = s._ranges["own"]
            s.fluid.pos[a:b].copy_(hpos[:b - a], non_blocking=True)
            s.fluid.vel[a:b].copy_(hvel[:b - a], non_blocking=True)
            return 24 * (b - a)

        down()
        torch.cuda.synchronize()
        k2 = max(3, args.steps // 2)
        f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h2d = d2h = 0
        f0.record()
        for _ in range(k2):
            h2d += up()
            s.step()
            d2h += down()
        f1.record()
        torch.cuda.synchronize()
        e2e = (f0.elapsed_time(f1) / k2, h2d / k2, d2h / k2)
    except RuntimeError as exc:
        if "skipped:" not in str(exc):
            # a rank that fails INSIDE the leg cannot tell the others (they wait for it in the next halo): take the job down
            # at once instead of letting it sit on the GPUs until the watchdog fires
            print(f"[bench] rank {rank}: e2e leg failed: {exc}", file=sys.stderr, flush=True)
            raise
        print(f"[bench] rank {rank}: e2e leg {exc}", file=sys.stderr, flush=True)   # agreed by all ranks: the line above stays valid
    t = torch.tensor([e2e[0] if e2e else -1.0, 0.0 if e2e else 1.0, e2e[1] if e2e else 0.0, e2e[2] if e2e else 0.0],
                     dtype=torch.float64, device=s.device)
    tmax = t.clone()
    dist.all_reduce(tmax, op=dist.ReduceOp.MAX)            # slowest rank; any failure flags the leg
    dist.all_reduce(t)                                      # bytes summed over ranks
    e2e_ms, e2e_failed = float(tmax[0].item()), bool(tmax[1].item() > 0)
    e2e_h2d, e2e_d2h = int(t[2].item()), int(t[3].item())
    comm = s.comm_s / (args.steps + (0 if e2e is None else max(3, args.steps // 2)))
    assembly_ms = s.assembly_ms() if s.mg is not None else None
    bytes_sent, msgs = s.comm_stats()
    strays = {"capacity_per_rank_and_step": s.stray_cap, "collected_per_rank_in_the_last_step": s.stray_counts(),
              "note": "particles that crossed >= 2 cell planes in one step are routed to every rank (include/sphk.h, Strays)"}
    transport = {None: "torch.distributed P2P", 0: "NCCL send/recv (native)", 1: "peer-memory mailboxes (CUDA IPC over NVLink) + NCCL candidates"}[getattr(s, "transport", None) if s.mg is not None else None]
    s.close()
    dist.destroy_process_group()
    if rank != 0:
        return None
    ms_step = float(ms.item()) / args.steps
    value = n / (ms_step * 1e-3)
    return {"metric": "particle-steps/sec (dam-break)", "value": value, "unit": "particle-steps/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": B.workload_name(scene_name, solver), "n_fluid": n, "n_boundary": int(sc.n_boundary),
                       "scene_init": "device-side (sphk_scene_fluid_block / sphk_scene_boundary_shell: no host particle arrays)" if sc.fluid is None else "host arrays",
                       "cells": list(sc.params.cell_size), "parallelism": f"x-slabs x{world}, halo = 1 cell plane, {transport}",
                       "per_gpu_particles_max": int(mx[0].item()), "load_imbalance": float(mx[0].item() * world / own[0].item()),
                       "l2": "inputs larger than L2 (packed records + neighbour list per rank > 50 MB L2); no flush"},
            "e2e": ({"value": value, "unit": "particle-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                     "note": "e2e leg failed on a rank; device-resident value repeated"} if e2e_failed else
                    {"value": n / (e2e_ms * 1e-3), "unit": "particle-steps/s", "ms_per_step": e2e_ms,
                     "h2d_bytes_per_step": e2e_h2d, "d2h_bytes_per_step": e2e_d2h, "steps": max(3, args.steps // 2),
                     "api": "SlabSystem.step() per rank; every step uploads the rank's owned pos+vel from pinned host buffers "
                            "and downloads pos+vel+density into them (bytes summed over ranks)",
                     "timer": "CUDA events on the compute stream (copies are enqueued on it), max over ranks"}),
            "parity_checked": bool(parity and parity["parity_checked"]), "max_rel_err": (parity or {}).get("max_rel_err"), "parity": parity,
            "gpu_launches": int(launches.item()), "strays": strays, "halo": {"assembly_ms_per_step_device": assembly_ms,
                                                           "assembly_note": "candidate exchange + search of [ghosts|owned] + plane offsets (host read) + count "
                                                                            "exchange + list build, CUDA events on rank 0; the rest of the step is sweeps + one halo kernel each",
                                                           "host_wall_seconds_per_step_in_begin_step": comm,
                                                           "bytes_sent_rank0_total": bytes_sent, "messages_rank0_total": msgs},
            "clocks": clocks}
