"""Sync-free training step on the fused C-ABI path (what reference train.py:159-185 does per step, plus
the optimiser PL runs after it and the every-16-steps occupancy refresh of train.py:160-163):

    [device RNG -> batch assembly] -> ngp_render_train_fwd -> ngp_nerf_loss_grad -> ngp_render_train_bwd
    -> [one NCCL all-reduce of the flat gradient buffer] -> ngp_adam_step (+fp16 re-cast, +grad zero)

All of it is stream-ordered launches with no host synchronisation, so `capture()` records it into one
CUDA graph. Parameters live in ONE flat fp32 buffer [xyz_encoder.params | rgb_net.params] (the
nn.Parameters of the NGP module are views into it, so state_dict()/checkpoints keep the reference's
keys and layouts); gradients, Adam moments and the fp16 working copy mirror that layout.

Data parallelism (reference train.py:269-272: DDP, one process per GPU, every rank draws its own
batch => weak scaling): a single `all_reduce(SUM)` over the flat gradient buffer per step, averaged
inside the Adam kernel (grad_mul = 1/world_size). The occupancy bitfield is refreshed by every rank
from identical parameters and then broadcast from rank 0 so all ranks march the same grid.
"""
import ctypes as C
import gc
import math

import torch

from . import _lib
from .models.networks import NGP, feat_save_bytes
from .models.rendering import MAX_SAMPLES, NEAR_DISTANCE


def allreduce_gradients(flat_grad, world_size, process_group=None):
    """The ONE collective of a data-parallel step: SUM all-reduce of the flat gradient buffer (the 1/N of
    DDP's mean is applied by the Adam kernel's grad_mul). Backend-agnostic (NCCL on GPUs, gloo in the CPU tests)."""
    if world_size > 1:
        import torch.distributed as dist
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=process_group)
    return flat_grad


def broadcast_occupancy(density_bitfield, world_size, process_group=None, src=0):
    """Occupancy policy: all ranks march rank `src`'s bitfield (the reference leaves this to DDP buffer sync)."""
    if world_size > 1:
        import torch.distributed as dist
        dist.broadcast(density_bitfield, src=src, group=process_group)
    return density_bitfield


def zero_shard(n_params, world_size, rank):
    """"zero" mode: (lo, hi, n_pad) -- the flat buffers are padded to n_pad = a multiple of 4*world so that every rank owns
    an equal, 16-byte aligned slice [rank*n_pad/world, (rank+1)*n_pad/world) of which [lo, hi) are real parameters"""
    q = 4 * world_size
    n_pad = (n_params + q - 1) // q * q
    shard = n_pad // world_size
    lo = min(rank * shard, n_params)
    hi = min(lo + shard, n_params)
    return lo, hi, n_pad


def zero_exchange(G_full, G_shard, Ph_full, shard_bounds, rank, world_size, process_group, adam_on_shard):
    """One optimiser step of the "zero" mode on the padded flat buffers: reduce_scatter(SUM) of the gradient into this rank's
    shard, clear the local gradient, `adam_on_shard(lo, hi, G_shard)` updates the owned parameters [lo, hi) (and writes their
    slice of the fp16 working copy Ph_full), all_gather of the working copy. Pure orchestration: the GPU trainer passes the
    CUDA Adam kernel, the gloo test a torch one."""
    import torch.distributed as dist
    lo, hi, n_pad = shard_bounds
    shard = n_pad // world_size
    dist.reduce_scatter_tensor(G_shard, G_full, op=dist.ReduceOp.SUM, group=process_group)
    G_full.zero_()
    if hi > lo:
        adam_on_shard(lo, hi, G_shard)
    mine = rank * shard  # (lo is clamped to n_params when a shard is all padding)
    dist.all_gather_into_tensor(Ph_full, Ph_full[mine:mine + shard], group=process_group)


def shard_range(n_items, world_size, rank):
    """contiguous shard [lo, hi) of n_items (test views / image rows) for `rank`; sizes differ by at most one"""
    base, extra = divmod(n_items, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


class CosineAnnealingLR:
    """The reference's learning-rate schedule (train.py:135-137): torch.optim.lr_scheduler.CosineAnnealingLR(opt,
    T_max=num_epochs, eta_min=lr/30), which pytorch-lightning steps once per EPOCH; a training epoch of the reference is
    1000 optimiser steps (datasets/base.py:17-19). So the rate is piecewise constant:
        lr(step) = eta_min + (lr0 - eta_min) * (1 + cos(pi * epoch / T_max)) / 2,   epoch = step // steps_per_epoch.
    Trainer(lr_schedule=...) writes it into the device-resident `lr` the Adam kernels read (stream-ordered fill, no sync,
    no graph re-capture)."""

    def __init__(self, base_lr, T_max=30, eta_min=None, steps_per_epoch=1000):
        self.base_lr = float(base_lr)
        self.T_max = int(T_max)
        self.eta_min = float(base_lr) / 30 if eta_min is None else float(eta_min)
        self.steps_per_epoch = int(steps_per_epoch)

    def lr_at_epoch(self, epoch):
        return self.eta_min + (self.base_lr - self.eta_min) * (1 + math.cos(math.pi * epoch / self.T_max)) / 2

    def lr_at_step(self, step):
        return self.lr_at_epoch(step // self.steps_per_epoch)


def log_ring_spans(first, n, rows):
    """The per-step log keeps step k in row k % rows of its ring. Returns the ring slices [lo, hi) that hold steps
    first .. first + n - 1, in step order (two slices when the range wraps). n may not exceed rows: older steps of the
    range would already be overwritten."""
    if n < 0 or rows < 1:
        raise ValueError("log_ring_spans: n must be >= 0 and rows >= 1, got n=%d rows=%d" % (n, rows))
    if n > rows:
        raise RuntimeError("log_ring_spans: %d steps do not fit a ring of %d rows" % (n, rows))
    spans, s = [], first
    while n > 0:
        lo = s % rows
        k = min(n, rows - lo)
        spans.append((lo, lo + k))
        s += k
        n -= k
    return spans


def log_rows_to_stats(rows, n_rays, lambda_opacity, lambda_distortion=0.0, live=True):
    """Decode rows of the per-step log ((n, 8) int32 numpy, the layout of ngp_train_log_step) into the dicts
    Trainer.stats() returns after that step -- the same formulas on the same fp32 values, so loss, mse, psnr and the
    sample counts are bitwise stats()'s -- plus 'step' (0-based index) and 'lr' (the fp32 rate the step's Adam used).
    lambda_opacity must be the value the kernels saw (Trainer.cfg.lambda_opacity); live: whether the trainer skips dead
    samples (bw_samples is rm_samples otherwise). With lambda_distortion > 0, 'distortion' is the mean of the step's
    distortion loss times lambda_distortion from a double sum (stats() takes torch's fp32 mean), and is part of 'loss'."""
    import numpy as np
    rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 8)
    f = rows.view(np.float32)
    out = []
    for r, x in zip(rows.tolist(), f.tolist()):
        n = n_rays
        mse = x[0] / (3 * n)
        loss = mse + lambda_opacity * x[1] / n
        d = dict(rm_samples=r[2], vr_samples=r[3], bw_samples=r[4] if live else r[2], mse=mse,
                 psnr=-10 * math.log10(max(mse, 1e-12)))
        if lambda_distortion > 0:
            d["distortion"] = lambda_distortion * (x[6] / n)
            loss += d["distortion"]
        d["loss"] = loss
        d["step"] = r[7]
        d["lr"] = x[5]
        out.append(d)
    return out


_SET_FIELDS = ("rays_o", "rays_d", "rgb_gt", "noise", "n_samples", "offsets", "counters", "ray_idx", "ts", "deltas", "bg")


class Trainer:
    def __init__(self, model: NGP, n_rays=8192, lr=1e-2, exp_step_factor=0.0, bg=(1.0, 1.0, 1.0), lambda_opacity=1e-3,
                 T_threshold=1e-4, betas=(0.9, 0.999), eps=1e-15, max_total_samples=None, update_interval=16,
                 warmup_steps=256, process_group=None, world_size=1, rank=0, seed=0, materialize_ws=False, ddp="nccl",
                 lambda_distortion=0.0, skip_dead_samples=True, fused_loss=True, random_bg=False, erode=False,
                 lr_schedule=None, pick_ahead=True, ray_sampling_strategy="all_images", log_rows=0):
        if int(log_rows) < 0:
            raise ValueError("Trainer: log_rows must be >= 0 (0 = no per-step log), got %r" % (log_rows,))
        if ray_sampling_strategy not in ("all_images", "same_image"):
            raise ValueError("Trainer: ray_sampling_strategy must be 'all_images' or 'same_image', got %r" % (ray_sampling_strategy,))
        self.ray_sampling_strategy = ray_sampling_strategy  # reference opt.py:34-39
        self.model = model
        self.pick_ahead = pick_ahead
        self._picked = None
        self._pick_stream = None
        dev = model.density_bitfield.device
        if dev.type != "cuda":
            raise RuntimeError("ngp_pl_b200.Trainer needs the model on a CUDA device (there is no CPU path)")
        self.dev = dev
        self.n_rays = int(n_rays)
        self.lr = float(lr)
        self.betas, self.eps = betas, float(eps)
        self.update_interval, self.warmup_steps = update_interval, warmup_steps
        self.pg, self.world_size, self.rank = process_group, int(world_size), int(rank)
        self.exp_step_factor = float(exp_step_factor)
        self.lambda_distortion = float(lambda_distortion)  # reference opt.py:25 --distortion_loss_w (0 = off)
        if self.lambda_distortion > 0:
            materialize_ws = True
        self.host_step = 0
        self.seed = seed
        # the distortion loss needs the per-sample weights between the compositing forward and backward: separate kernels
        self.fused_loss = bool(fused_loss) and not (lambda_distortion > 0) and not materialize_ws
        # "nccl": all_reduce of the flat gradient + full Adam on every rank (what the reference's DDP does);
        # "zero": NCCL reduce_scatter of the gradient + Adam on this rank's 1/N shard + all_gather of the fp16 working
        #         copy: 3/4 of all_reduce's traffic ((N-1)/N * (4+2) instead of 2*(N-1)/N * 4 bytes per parameter) and 1/N of
        #         the optimiser's HBM traffic;
        # "p2p" : the same algorithm as ONE self-synchronising kernel over NVLink peer memory (ngp_adam_step_fused: flag
        #         barriers inside the kernel, captured into the step's CUDA graph, gradient buffers alternate so the clear
        #         of the next one rides in the same kernel);
        # "nvls": "p2p" with the NVSwitch doing the sum / the replication (multimem.ld_reduce / multimem.st on the
        #         multicast mapping of the symmetric buffers);
        # "p2p_host": round 1's variant of "p2p" (host-launched barriers around ngp_adam_step_p2p), kept for comparison
        self.ddp = ddp if self.world_size > 1 else "none"
        self.random_bg = bool(random_bg)   # reference rendering.py:153-161 (one random colour per training batch)
        self.erode = bool(erode)           # reference networks.py:258-260 / train.py:163 (needs model.count_grid)
        self.lr_schedule = lr_schedule     # e.g. CosineAnnealingLR(lr, T_max=30, steps_per_epoch=1000)
        self._n_gbuf = 2 if self.ddp in ("p2p", "nvls") else 1
        self._gcur = 0
        L = _lib.lib()

        # ---- flat parameter / gradient / optimiser state --------------------------------------------------
        pe, pr = model.xyz_encoder.params, model.rgb_net.params
        self.n_enc, self.n_rgb = pe.numel(), pr.numel()
        n = self.n_enc + self.n_rgb
        self.n_params = n
        with torch.cuda.device(dev):
            self.P = torch.empty(n, device=dev, dtype=torch.float32)
            self.P[:self.n_enc].copy_(pe.data)
            self.P[self.n_enc:].copy_(pr.data)
            pe.data = self.P[:self.n_enc]
            pr.data = self.P[self.n_enc:]
            if self.ddp in ("p2p", "nvls", "p2p_host"):
                # gradient buffer(s), fp16 working copy and the barrier flags live in symmetric (peer-mapped) memory
                import torch.distributed as dist
                import torch.distributed._symmetric_memory as symm_mem
                if n % 4:
                    raise RuntimeError("the fused exchange needs a parameter count that is a multiple of 4")
                grp = self.pg if self.pg is not None else dist.group.WORLD
                W = self.world_size
                self._G2 = symm_mem.empty(self._n_gbuf * n, dtype=torch.float32, device=dev)
                self._G2.zero_()
                self._Gs = [self._G2[b * n:(b + 1) * n] for b in range(self._n_gbuf)]
                self.Ph = symm_mem.empty(n, dtype=torch.float16, device=dev)
                self._flags = symm_mem.empty(64, dtype=torch.int32, device=dev)
                self._flags.zero_()
                self._sync = torch.zeros(8, device=dev, dtype=torch.int32)
                self.hG = symm_mem.rendezvous(self._G2, grp)
                self.hPh = symm_mem.rendezvous(self.Ph, grp)
                self.hFl = symm_mem.rendezvous(self._flags, grp)
                self.peer_Gs = [(C.c_uint64 * W)(*[int(p) + 4 * n * b for p in self.hG.buffer_ptrs]) for b in range(self._n_gbuf)]
                self.peer_G = self.peer_Gs[0]
                self.peer_Ph = (C.c_uint64 * W)(*[int(p) for p in self.hPh.buffer_ptrs])
                self.peer_flags = (C.c_uint64 * W)(*[int(p) for p in self.hFl.buffer_ptrs])
                self.mc_Gs, self.mc_Ph = [0] * self._n_gbuf, 0
                if self.ddp == "nvls":
                    mg, mp = int(getattr(self.hG, "multicast_ptr", 0) or 0), int(getattr(self.hPh, "multicast_ptr", 0) or 0)
                    if not mg or not mp:
                        raise RuntimeError("ddp='nvls': the symmetric allocations have no multicast (NVLS) mapping on this system")
                    self.mc_Gs = [mg + 4 * n * b for b in range(self._n_gbuf)]
                    self.mc_Ph = mp
                torch.cuda.synchronize(dev)
                dist.barrier(group=self.pg)  # every rank's flags / gradients are zero before anyone's first exchange
            elif self.ddp == "zero":
                # equal shards for reduce_scatter / all_gather: pad the flat buffers to a multiple of 4 * world
                lo, hi, n_pad = zero_shard(n, self.world_size, self.rank)
                self._zero = (lo, hi, n_pad)
                self.G_full = torch.zeros(n_pad, device=dev, dtype=torch.float32)
                self.Ph_full = torch.zeros(n_pad, device=dev, dtype=torch.float16)
                self._Gs, self.Ph = [self.G_full[:n]], self.Ph_full[:n]
                self.G_shard = torch.zeros(n_pad // self.world_size, device=dev, dtype=torch.float32)
            else:
                self._Gs = [torch.zeros(n, device=dev, dtype=torch.float32)]
                self.Ph = torch.empty(n, device=dev, dtype=torch.float16)
            self.M = torch.zeros(n, device=dev, dtype=torch.float32)
            self.V = torch.zeros(n, device=dev, dtype=torch.float32)
            _lib.check(L.ngp_cast_params(self.P.data_ptr(), self.Ph.data_ptr(), n, self._st()), "cast_params")
            # the module-level API (NGP.forward / density / render) must see the weights this trainer updates
            from .tcnn import _FixedHalf
            model.xyz_encoder._half = _FixedHalf(self.Ph[:self.n_enc])
            model.rgb_net._half = _FixedHalf(self.Ph[self.n_enc:])
            self.lr_dev = torch.full((1,), self.lr, device=dev, dtype=torch.float32)
            self.step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
            # per-step log (drain_log): ring of log_rows rows written on the device by ngp_train_log_step
            self.log_rows = int(log_rows)
            self.log_ring = torch.zeros(self.log_rows, 8, device=dev, dtype=torch.int32) if self.log_rows else None
            self._log_next = 0        # first step not yet enqueued for a copy
            self._log_pending = []    # (first step, n, pinned rows, copy-done event), oldest first
            self._log_stream = None
            self._log_quiet = False

            # ---- network descriptor pointing at the flat fp16 copy -----------------------------------------
            net = _lib.NgpNet()
            net.enc_params_h = self.Ph.data_ptr()
            net.rgb_params_h = self.Ph[self.n_enc:].data_ptr()
            net.meta = model.xyz_encoder.meta
            for k in range(3):
                net.xyz_min[k] = model._xyz_min_host[k]
                net.xyz_max[k] = model._xyz_max_host[k]
            net.rgb_act = model.rgb_net.rgb_act
            self.net = net

            # ---- step configuration -------------------------------------------------------------------------
            cfg = _lib.NgpTrainCfg()
            cfg.n_rays = self.n_rays
            cfg.cascades = model.cascades
            cfg.grid_size = model.grid_size
            cfg.max_samples = MAX_SAMPLES
            cfg.scale = float(model.scale)
            cfg.exp_step_factor = self.exp_step_factor
            cfg.T_threshold = float(T_threshold)
            cfg.near_distance = NEAR_DISTANCE
            c, h = model.center.flatten().tolist(), model.half_size.flatten().tolist()
            for k in range(3):
                cfg.center[k], cfg.half_size[k], cfg.bg[k] = c[k], h[k], float(bg[k])
            cfg.lambda_opacity = float(lambda_opacity)
            cap = int(max_total_samples) if max_total_samples else self.n_rays * MAX_SAMPLES
            cfg.max_total_samples = cap
            self.cfg = cfg
            self.capacity = cap

            # ---- buffers ------------------------------------------------------------------------------------
            f32 = dict(device=dev, dtype=torch.float32)
            i32 = dict(device=dev, dtype=torch.int32)
            N = self.n_rays
            # Two sets of everything the batch assembly + march WRITE and the network step READS (rays, jitter, per-ray
            # counts, compacted samples, counters): the next step's batch is marched into the other set while this
            # step's network forward / backward / optimiser run (capture(): deep pipeline).
            self._sets = []
            for _ in range(2):
                self._sets.append(dict(
                    rays_o=torch.zeros(N, 3, **f32), rays_d=torch.zeros(N, 3, **f32), rgb_gt=torch.zeros(N, 3, **f32),
                    noise=torch.zeros(N, **f32), n_samples=torch.zeros(N, **i32), offsets=torch.zeros(N, **i32),
                    counters=torch.zeros(8, **i32), ray_idx=torch.empty(cap, **i32), ts=torch.empty(cap, **f32),
                    deltas=torch.empty(cap, **f32), bg=torch.tensor([float(v) for v in bg], **f32)))
            self._cur = 0
            self.stage_t = torch.empty(N * MAX_SAMPLES, **f32)
            self.stage_dt = torch.empty(N * MAX_SAMPLES, **f32)
            self.rgb = torch.zeros(N, 3, **f32)
            self.opacity = torch.zeros(N, **f32)
            self.depth = torch.zeros(N, **f32)
            self.sigmas = torch.empty(cap, **f32)
            self.rgbs = torch.empty(cap, 3, **f32)
            self.ws = torch.empty(cap, **f32) if materialize_ws else None
            self.dsigmas = torch.empty(cap, **f32)
            self.drgbs = torch.empty(cap, 3, **f32)
            # samples past a ray's termination get exactly zero gradient: the backward visits only the others
            self.live_idx = torch.empty(cap, **i32) if skip_dead_samples else None
            self.feat_save = torch.empty(feat_save_bytes(cap), device=dev, dtype=torch.uint8)
            self.scalars = torch.zeros(8, **f32)
            self.dL_drgb = torch.zeros(N, 3, **f32)
            self.dL_dopacity = torch.zeros(N, **f32)
            if self.lambda_distortion > 0:
                # DistortionLoss (reference losses.py:6-37) on the fused path: per-sample scans + dL/dws
                self.rays_a = torch.zeros(N, 3, device=dev, dtype=torch.int64)
                self.rays_a[:, 0] = torch.arange(N, device=dev)
                self.dist_loss = torch.zeros(N, **f32)
                self.dist_dL = torch.full((N,), self.lambda_distortion / N, **f32)  # d(mean(lambda*loss))/dloss
                self.ws_inc = torch.empty(cap, **f32)
                self.wts_inc = torch.empty(cap, **f32)
                self.dL_dws = torch.zeros(cap, **f32)
            scan_bytes = L.ngp_train_scan_temp_bytes(N)
            self.scan_temp = torch.zeros(scan_bytes, device=dev, dtype=torch.uint8)  # march accumulators: zero once
            bwd_bytes = L.ngp_net_backward_workspace(cap)
            self.bwd_ws = torch.empty(bwd_bytes, device=dev, dtype=torch.uint8)
            for st_ in self._sets:
                b = _lib.NgpTrainBuffers()
                for name in _SET_FIELDS:
                    if name not in ("rgb_gt", "bg"):
                        setattr(b, name, st_[name].data_ptr())
                for name in ("stage_t", "stage_dt", "rgb", "opacity", "depth", "sigmas", "rgbs", "dsigmas", "drgbs",
                             "feat_save", "scalars", "scan_temp"):
                    setattr(b, name, getattr(self, name).data_ptr())
                b.ws = self.ws.data_ptr() if self.ws is not None else None
                b.live_idx = self.live_idx.data_ptr() if self.live_idx is not None else None
                b.density_bitfield = model.density_bitfield.data_ptr()
                b.scan_temp_bytes = scan_bytes
                b.bwd_workspace = self.bwd_ws.data_ptr()
                b.bwd_workspace_bytes = bwd_bytes
                b.bg_dev = st_["bg"].data_ptr() if self.random_bg else None
                st_["buf"] = b

            # ---- occupancy grid ----------------------------------------------------------------------------
            G3 = model.grid_size ** 3
            if not hasattr(model, "density_grid"):
                model.register_buffer("density_grid", torch.zeros(model.cascades, G3, **f32))
            ws_bytes = L.ngp_update_grid_workspace(model.cascades, model.grid_size)
            self.grid_ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            self.gen = torch.Generator(device=dev)
            self.gen.manual_seed(seed + 1000 * self.rank)
        # model.load_state_dict(...) writes the fp32 parameters behind the kernels' back: refresh the fp16 working copy
        self._load_hook = model.register_load_state_dict_post_hook(lambda module, incompatible: self.sync_params())
        self.graph = False
        self.graph_launches = 0
        self._graph_nodes = {}
        self._graph_samples = None
        self._premarched = False
        self._staged = None
        self._inflight = False
        self.bank = None

    # ------------------------------------------------------------------------------------------------------
    def __getattr__(self, name):
        # rays_o, rays_d, rgb_gt, noise, n_samples, offsets, counters, ray_idx, ts, deltas, buf: those of the set the
        # current / last completed step works on
        if name in _SET_FIELDS or name == "buf":
            sets = self.__dict__.get("_sets")
            if sets:
                return sets[self.__dict__.get("_cur", 0)][name]
        raise AttributeError(name)

    def _st(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    @property
    def G(self):
        """the flat fp32 gradient buffer the step in flight accumulates into (the fused exchange alternates between two)"""
        return self._Gs[self._gcur]

    def set_lr(self, lr):
        self.lr = float(lr)
        self.lr_dev.fill_(float(lr))  # stream-ordered, no sync; the Adam kernels read lr from the device

    def sync_params(self):
        """Call after writing the fp32 parameters from outside (load_state_dict, p.data.copy_, EMA swap...): refreshes the
        fp16 working copy every kernel reads. In the sharded modes every rank must call it with identical parameters."""
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().ngp_cast_params(self.P.data_ptr(), self.Ph.data_ptr(), self.n_params, self._st()), "cast_params")
        if self.world_size > 1 and self.ddp in ("p2p", "nvls", "p2p_host", "zero"):
            import torch.distributed as dist
            torch.cuda.synchronize(self.dev)
            dist.barrier(group=self.pg)

    def _refresh_seed(self, step):
        return (self.seed * 2654435761 + step * 40503 + 12345) & 0xffffffff

    def _pick_key(self, step, density_threshold, warmup):
        g = self.model.density_grid
        return (self._refresh_seed(step), float(density_threshold), bool(warmup), g.data_ptr(), g._version)

    def _launch_pick(self, step, density_threshold, warmup, stream):
        m = self.model
        rc = _lib.lib().ngp_update_density_grid_pick(
            m.density_grid.data_ptr(), m.cascades, m.grid_size, float(m.scale), float(density_threshold), int(bool(warmup)),
            self._refresh_seed(step), self.grid_ws.data_ptr(), self.grid_ws.numel(), stream.cuda_stream)
        _lib.check(rc, "update_density_grid_pick")

    def update_density_grid(self, density_threshold=0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=False, decay=0.95, erode=None):
        """device-side equivalent of NGP.update_density_grid (reference networks.py:240-269); no host sync.
        erode (default: the constructor's): per-cell decay from model.count_grid (mark_invisible_cells), networks.py:258-260

        The refresh has a weight-independent half (which cells to re-evaluate -- it reads the OLD grid -- sorted, a jittered
        point in each: ngp_update_density_grid_pick) and a weight-dependent half (density at those points, merge, threshold,
        bitfield: ..._eval). With pick_ahead (default) the first half of the NEXT refresh is launched on its own stream as
        soon as this refresh is done, so that it runs under the training steps in between and only the second half sits
        between two steps; a pick is reused only if seed, threshold, warm-up flag and the grid tensor (address and torch
        version counter) are what it was made for, otherwise it is redone in line."""
        m = self.model
        erode = self.erode if erode is None else erode
        count = None
        if erode:
            if not hasattr(m, "count_grid"):
                raise RuntimeError("erode=True needs model.count_grid: call model.mark_invisible_cells(K, poses, img_wh) first")
            count = m.count_grid.data_ptr()
        with torch.cuda.device(self.dev):
            main = torch.cuda.current_stream(self.dev)
            key = self._pick_key(self.host_step, density_threshold, warmup)
            picked, self._picked = self._picked, None
            if picked is not None:
                main.wait_event(picked[1])  # also when stale: it may still be writing the workspace
            if picked is None or picked[0] != key:
                self._launch_pick(self.host_step, density_threshold, warmup, main)
            rc = _lib.lib().ngp_update_density_grid_eval(
                C.byref(self.net), m.density_grid.data_ptr(), m.density_bitfield.data_ptr(), count, m.cascades, m.grid_size,
                float(density_threshold), int(bool(warmup)), float(decay), self.grid_ws.data_ptr(), self.grid_ws.numel(),
                main.cuda_stream)
            _lib.check(rc, "update_density_grid_eval")
            broadcast_occupancy(m.density_bitfield, self.world_size, self.pg)
            if self.pick_ahead and not torch.cuda.is_current_stream_capturing():
                if self._pick_stream is None:
                    self._pick_stream = torch.cuda.Stream(self.dev)
                    self.grid_ws.record_stream(self._pick_stream)
                nxt = self.host_step + self.update_interval
                warm_next = nxt < self.warmup_steps
                done = torch.cuda.Event()
                done.record(main)
                self._pick_stream.wait_event(done)
                m.density_grid.record_stream(self._pick_stream)  # read there: keep its memory from being recycled under the pick
                self._launch_pick(nxt, density_threshold, warm_next, self._pick_stream)
                ev = torch.cuda.Event()
                ev.record(self._pick_stream)
                self._picked = (self._pick_key(nxt, density_threshold, warm_next), ev)

    # ---- pieces of one step (all asynchronous) -------------------------------------------------------------
    def attach_bank(self, bank):
        """bank: any object with device tensors `poses` (n,3,4) float32, `directions` (hw,3) float32 and `rgb` (n,hw,3)
        uint8 (read as v/255) or float32, all contiguous on the trainer's device -- synth.RayBank, datasets.load_scene().
        Anything else raises."""
        poses, dirs, rgb = (getattr(bank, k, None) for k in ("poses", "directions", "rgb"))
        for name, t in (("poses", poses), ("directions", dirs), ("rgb", rgb)):
            if not isinstance(t, torch.Tensor):
                raise RuntimeError("Trainer.attach_bank: bank.%s must be a tensor, got %s" % (name, type(t).__name__))
            if t.device != self.dev:
                raise RuntimeError("Trainer.attach_bank: bank.%s is on %s, the trainer on %s" % (name, t.device, self.dev))
            if not t.is_contiguous():
                raise RuntimeError("Trainer.attach_bank: bank.%s must be contiguous" % name)
        n, hw = poses.shape[0] if poses.dim() == 3 else -1, dirs.shape[0]
        if poses.dtype != torch.float32 or poses.dim() != 3 or tuple(poses.shape[1:]) != (3, 4) or n < 1:
            raise RuntimeError("Trainer.attach_bank: bank.poses must be float32 (n,3,4), got %s %s" % (poses.dtype, tuple(poses.shape)))
        if dirs.dtype != torch.float32 or dirs.dim() != 2 or dirs.shape[1] != 3 or hw < 1:
            raise RuntimeError("Trainer.attach_bank: bank.directions must be float32 (hw,3), got %s %s" % (dirs.dtype, tuple(dirs.shape)))
        if rgb.dtype not in (torch.uint8, torch.float32) or tuple(rgb.shape) != (n, hw, 3):
            raise RuntimeError("Trainer.attach_bank: bank.rgb must be uint8 or float32 (%d,%d,3), got %s %s"
                               % (n, hw, rgb.dtype, tuple(rgb.shape)))
        self.bank = bank

    def sample_batch(self):
        """random (image, pixel) pairs with replacement (reference datasets/base.py:22-30; with 'same_image' one image per
        batch) + ray assembly + the march's start jitter, one kernel with a device-side counter-based generator (one
        stream per buffer set)"""
        bk = self.bank
        rc = _lib.lib().ngp_sample_rays_ex(
            bk.poses.data_ptr(), bk.directions.data_ptr(), bk.rgb.data_ptr(), int(bk.rgb.dtype == torch.float32),
            int(self.ray_sampling_strategy == "same_image"), bk.poses.shape[0], bk.directions.shape[0], self.n_rays,
            (self.seed * 2654435761 + 97 * self.rank) & 0xffffffff, self._cur, self.counters[6:].data_ptr(),
            self.rays_o.data_ptr(), self.rays_d.data_ptr(), self.rgb_gt.data_ptr(), self.noise.data_ptr(), self._st())
        _lib.check(rc, "sample_rays")

    def set_batch(self, rays_o, rays_d, rgb_gt):
        self.rays_o.copy_(rays_o, non_blocking=True)
        self.rays_d.copy_(rays_d, non_blocking=True)
        self.rgb_gt.copy_(rgb_gt, non_blocking=True)

    def stage_batch(self, rays_o, rays_d, rgb_gt):
        """Prefetch for host-fed training (train_step(sample=False)): copy the NEXT step's batch (pinned host or device
        tensors) into the other buffer set and march it on the side stream, under whatever step is in flight. The next
        train_step(sample=False) consumes it. Falls back to set_batch() when the step is not graph-captured."""
        if not (self.graph and self._graph_samples is False):
            return self.set_batch(rays_o, rays_d, rgb_gt)
        nxt = 1 - self._cur if (self._inflight or self._premarched) else self._cur
        st_ = self._sets[nxt]
        self._side.wait_event(self._ev_set[nxt])  # the set's last reader (the compute two steps back)
        with torch.cuda.stream(self._side):
            st_["rays_o"].copy_(rays_o, non_blocking=True)
            st_["rays_d"].copy_(rays_d, non_blocking=True)
            st_["rgb_gt"].copy_(rgb_gt, non_blocking=True)
            if self.host_step % self.update_interval != 0:
                # (ahead of a refresh step the march would read the bitfield while the refresh rewrites it, and its result
                # would be discarded anyway: train_step marches after the refresh)
                self._replay(self.g_prepare[nxt])
        self._staged = nxt

    def march(self, jitter=True):
        """first half of the forward: start jitter + AABB + march + segment allocation (independent of the weights)"""
        if jitter:
            self.noise.uniform_(0, 1, generator=self.gen)
        if self.random_bg:
            self.bg.uniform_(0, 1, generator=self.gen)  # one colour per batch (reference rendering.py:156)
        _lib.check(_lib.lib().ngp_render_train_march(C.byref(self.cfg), C.byref(self.buf), self._st()), "render_train_march")

    def network(self):
        """second half of the forward: fused network kernel on the marched samples + ragged compositing"""
        _lib.check(_lib.lib().ngp_render_train_net(C.byref(self.net), C.byref(self.cfg), C.byref(self.buf), self._st()),
                   "render_train_net")

    def forward(self):
        self.march()
        self.network()

    def loss_backward(self):
        L = _lib.lib()
        self.scalars[2:4].zero_()
        _lib.check(L.ngp_nerf_loss_grad(C.byref(self.cfg), C.byref(self.buf), self.rgb_gt.data_ptr(),
                                        self.dL_drgb.data_ptr(), self.dL_dopacity.data_ptr(), self._st()), "nerf_loss_grad")
        dws = None
        if self.lambda_distortion > 0:
            self.rays_a[:, 1] = self.offsets
            self.rays_a[:, 2] = self.n_samples
            N, cap = self.n_rays, self.capacity
            _lib.check(L.ngp_distortion_loss_fw(self.ws.data_ptr(), self.deltas.data_ptr(), self.ts.data_ptr(),
                                                self.rays_a.data_ptr(), N, cap, self.dist_loss.data_ptr(),
                                                self.ws_inc.data_ptr(), self.wts_inc.data_ptr(), self._st()), "distortion_fw")
            _lib.check(L.ngp_distortion_loss_bw(self.dist_dL.data_ptr(), self.ws_inc.data_ptr(), self.wts_inc.data_ptr(),
                                                self.ws.data_ptr(), self.deltas.data_ptr(), self.ts.data_ptr(),
                                                self.rays_a.data_ptr(), N, cap, self.dL_dws.data_ptr(), self._st()), "distortion_bw")
            dws = self.dL_dws.data_ptr()
        _lib.check(L.ngp_render_train_bwd(C.byref(self.net), C.byref(self.cfg), C.byref(self.buf), self.dL_drgb.data_ptr(),
                                          self.dL_dopacity.data_ptr(), None, dws, self.G.data_ptr(),
                                          self.G[self.n_enc:].data_ptr(), self._st()), "render_train_bwd")

    def allreduce(self):
        if self.ddp == "nccl":
            allreduce_gradients(self.G, self.world_size, self.pg)

    def optimizer_step(self):
        """gradient exchange (N > 1) + Adam + fp16 re-cast + clearing of the gradient buffer the next step uses"""
        if self.ddp in ("p2p", "nvls"):
            self._launch_fused()
            self._gcur ^= 1
            return
        if self.ddp == "p2p_host":
            return self._optimizer_step_p2p_host()
        if self.ddp == "zero":
            return self._optimizer_step_zero()
        rc = _lib.lib().ngp_adam_step(self.P.data_ptr(), self.G.data_ptr(), self.M.data_ptr(), self.V.data_ptr(),
                                      self.Ph.data_ptr(), self.n_params, self.lr_dev.data_ptr(), self.step_dev.data_ptr(),
                                      self.betas[0], self.betas[1], self.eps, 1.0 / self.world_size, 1, self._st())
        _lib.check(rc, "adam_step")

    def _optimizer_step_zero(self):
        """reduce_scatter(grad) -> Adam on the owned shard (writes its slice of the fp16 copy) -> all_gather(fp16 copy)"""
        def adam_on_shard(lo, hi, g_shard):
            rc = _lib.lib().ngp_adam_step(self.P[lo:].data_ptr(), g_shard.data_ptr(), self.M[lo:].data_ptr(),
                                          self.V[lo:].data_ptr(), self.Ph_full[lo:].data_ptr(), hi - lo, self.lr_dev.data_ptr(),
                                          self.step_dev.data_ptr(), self.betas[0], self.betas[1], self.eps,
                                          1.0 / self.world_size, 1, self._st())
            _lib.check(rc, "adam_step")
        zero_exchange(self.G_full, self.G_shard, self.Ph_full, self._zero, self.rank, self.world_size, self.pg, adam_on_shard)

    def _launch_fused(self):
        """ONE kernel: start barrier -> reduce-scatter + sharded Adam + all-gather over NVLink (peer loads/stores or
        multimem) + clear of the other gradient buffer -> end barrier (ngp_adam_step_fused); graph-capturable"""
        b = self._gcur
        rc = _lib.lib().ngp_adam_step_fused(self.world_size, self.rank, self.peer_Gs[b], self.peer_Ph, self.peer_flags,
                                            self.mc_Gs[b], self.mc_Ph, self.P.data_ptr(), self.M.data_ptr(), self.V.data_ptr(),
                                            self.n_params, self._Gs[1 - b].data_ptr(), self._sync.data_ptr(),
                                            self.lr_dev.data_ptr(), self.step_dev.data_ptr(), self.betas[0], self.betas[1],
                                            self.eps, 1, self._st())
        _lib.check(rc, "adam_step_fused")

    def check_exchange(self):
        """raises if a fused exchange ever timed out waiting for a peer (synchronises)"""
        if self.ddp in ("p2p", "nvls") and int(self._sync[2].item()) != 0:
            raise RuntimeError("ngp_adam_step_fused: a peer did not arrive at a barrier within the timeout")

    def _optimizer_step_p2p_host(self):
        """round 1: barrier -> reduce-scatter + sharded Adam + all-gather kernel -> barrier -> clear own gradients"""
        self.hG.barrier(channel=0)
        rc = _lib.lib().ngp_adam_step_p2p(self.world_size, self.rank, self.peer_G, self.P.data_ptr(), self.M.data_ptr(),
                                          self.V.data_ptr(), self.peer_Ph, self.n_params, self.lr_dev.data_ptr(),
                                          self.step_dev.data_ptr(), self.betas[0], self.betas[1], self.eps, 1, self._st())
        _lib.check(rc, "adam_step_p2p")
        self.hG.barrier(channel=0)
        self.G.zero_()

    def shard_bounds(self, rank=None):
        """[lo, hi) element range of the parameters whose fp32 master / Adam state `rank` owns in the sharded modes"""
        r = self.rank if rank is None else rank
        if self.ddp == "zero":
            return zero_shard(self.n_params, self.world_size, r)[:2]
        lo4, hi4 = shard_range(self.n_params // 4, self.world_size, r)
        return 4 * lo4, 4 * hi4

    def gather_master_params(self):
        """the sharded modes keep the fp32 master copy of each shard on its owner only: broadcast every shard so that
        state_dict() / checkpoints are complete on every rank (call before saving; synchronises)."""
        if self.ddp not in ("p2p", "nvls", "p2p_host", "zero"):
            return
        import torch.distributed as dist
        for r in range(self.world_size):
            lo, hi = self.shard_bounds(r)
            dist.broadcast(self.P[lo:hi], src=r, group=self.pg)

    # ---- one optimiser step ----------------------------------------------------------------------------------
    def _prepare(self, sample):
        if sample:
            self.sample_batch()  # draws the jitter too
        self.march(jitter=not sample)

    def _compute(self):
        if self.fused_loss:
            # plain NeRFLoss: compositing forward + loss + compositing backward are one kernel (ngp_render_train_step)
            _lib.check(_lib.lib().ngp_render_train_step(C.byref(self.net), C.byref(self.cfg), C.byref(self.buf),
                                                        self.rgb_gt.data_ptr(), self.G.data_ptr(),
                                                        self.G[self.n_enc:].data_ptr(), self._st()), "render_train_step")
            return
        self.network()
        self.loss_backward()

    def _update(self):
        self.allreduce()
        self.optimizer_step()
        self._log_step()

    def _log_step(self):
        """with log_rows > 0: the step's row of the log ring, after the optimiser (which advanced step_dev) on the current
        stream; nothing at all otherwise"""
        if self.log_ring is None or self._log_quiet:
            return
        dist = self.dist_loss if self.lambda_distortion > 0 else None
        rc = _lib.lib().ngp_train_log_step(self.scalars.data_ptr(), self.counters.data_ptr(), self.lr_dev.data_ptr(),
                                           self.step_dev.data_ptr(), None if dist is None else dist.data_ptr(),
                                           0 if dist is None else dist.numel(), self.log_ring.data_ptr(), self.log_rows,
                                           self._st())
        _lib.check(rc, "train_log_step")

    def _step_body(self, sample):
        self._prepare(sample)
        self._compute()
        self._update()

    def _replay(self, g):
        self.graph_launches += self._graph_nodes.get(id(g), 0)
        g.replay()

    def launch_count(self):
        """kernel launches of libngp_b200 issued for this process so far: eager ones (ngp_launch_count, which also counted
        every launch recorded while capturing) + recorded launches x graph replays"""
        return int(_lib.lib().ngp_launch_count()) + self.graph_launches

    def _capture_graph(self, fn):
        g = torch.cuda.CUDAGraph()
        g.register_generator_state(self.gen)
        n0 = int(_lib.lib().ngp_launch_count())
        # No automatic garbage collection while capturing: torch.cuda.graph no longer collects before it begins, so a
        # dead object cycle holding CUDA graphs (a deleted Trainer's) could be collected in the middle of the capture,
        # where destroying a graph is not permitted and invalidates the capture. The cycle is collected afterwards.
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(g):
                fn()
        finally:
            if gc_was_enabled:
                gc.enable()
        self._graph_nodes[id(g)] = int(_lib.lib().ngp_launch_count()) - n0
        return g

    def capture(self, sample=True):
        """Record the step into CUDA graphs, one [prepare, compute] pair per buffer set plus the optimiser:
            g_prepare[i]    = [batch assembly (k_sample_rays), AABB + march + segment allocation]   -> writes set i
            g_compute[i][b] = [network fwd, compositing, NeRFLoss, compositing bwd, loss scale, MLP bwd, scatter]
                              reads set i, accumulates into gradient buffer b
            g_update[b]     = [Adam], or for N > 1 the self-synchronising exchange kernel reducing buffer b and clearing
                              buffer 1-b (the NCCL modes launch their collectives eagerly)
            g_step[i][b]    = g_compute[i][b] + g_update[b] as ONE graph, where no collective sits between them (one GPU,
                              "p2p", "nvls"): the kernels of the chain are programmatic dependents of each other
                              (common.cuh), and a graph boundary would drain the GPU between the scatter and the optimiser.
                              An external event-record node after the scatter marks set i as read (_ev_set[i]).
        train_step() replays g_step, or the split pair when an after_backward hook needs the boundary.
        The front of a step (batch assembly + march) depends on the rays, the jitter and the occupancy bitfield but
        NOT on the weights, so train_step() replays the NEXT step's g_prepare into the other buffer set on a side
        stream while this step's compute and optimiser run on the main stream (except across an occupancy refresh,
        whose new bitfield the next march must see -- the reference's ordering, train.py:160-163)."""
        dev = self.dev
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        state = [self.P, self.M, self.V, self.Ph, self.step_dev] + list(self._Gs)
        with torch.cuda.stream(s):
            # one eager run so lazy initialisation (cudaFuncSetAttribute, NCCL / symmetric-memory setup) is done
            saved = [t.clone() for t in state]
            gcur = self._gcur
            self._log_quiet = True  # a step that is undone below writes no log row
            try:
                self._step_body(sample)
            finally:
                self._log_quiet = False
            if self.ddp == "p2p_host":
                self.hG.barrier(channel=0)
            for t, v in zip(state, saved):
                t.copy_(v)
            self._gcur = gcur
            if self.ddp == "p2p_host":
                self.hG.barrier(channel=0)
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        self.g_prepare, self.g_compute, self.g_update = [], [], None
        keep = (self._cur, self._gcur)
        for i in range(2):
            self._cur = i
            self.g_prepare.append(self._capture_graph(lambda: self._prepare(sample)))
            per_buf = []
            for b in range(self._n_gbuf):
                self._gcur = b
                per_buf.append(self._capture_graph(self._compute))
            self.g_compute.append(per_buf)
        if self.ddp in ("p2p", "nvls"):
            self.g_update = []
            for b in range(self._n_gbuf):
                self._gcur = b
                self.g_update.append(self._capture_graph(self._launch_fused))
        elif self.ddp not in ("p2p_host", "zero"):
            self._gcur = 0
            self.g_update = [self._capture_graph(self.optimizer_step)]
        # the moment set i's last reader (a step's compute) is done: the next march into set i waits for it
        self._ev_set = [torch.cuda.Event(external=True) for _ in range(2)]
        self.g_step = None
        if self.ddp in ("none", "p2p", "nvls"):
            fork = torch.cuda.Stream(dev)
            self.g_step = []
            for i in range(2):
                self._cur = i
                per_buf = []
                for b in range(self._n_gbuf):
                    self._gcur = b
                    per_buf.append(self._capture_graph(lambda: self._compute_update(fork)))
                self.g_step.append(per_buf)
        self._cur, self._gcur = keep
        self.graph = True
        self._graph_samples = sample
        self._side = torch.cuda.Stream(dev)
        self._staged = None
        self._inflight = False
        self._premarched = False

    def _compute_update(self, fork):
        """what g_step records: the compute, then the optimiser straight after the scatter on the main stream; the event
        that set _cur is read hangs off the scatter on a forked branch (`fork`), so that no graph node sits between the
        scatter and the optimiser's kernel"""
        main = torch.cuda.current_stream(self.dev)
        self._compute()
        fork.wait_stream(main)
        self._ev_set[self._cur].record(fork)
        if self.ddp in ("p2p", "nvls"):
            self._launch_fused()
        else:
            self.optimizer_step()
        self._log_step()
        main.wait_stream(fork)

    def _graph_compute_update(self, after_backward):
        """the compute and the optimiser of a captured step on the main stream; _ev_set[_cur] is recorded once the compute
        is done"""
        if after_backward is None and self.g_step is not None:
            self._replay(self.g_step[self._cur][self._gcur])
            if self._n_gbuf == 2:
                self._gcur ^= 1
            return
        self._replay(self.g_compute[self._cur][self._gcur])
        if after_backward is not None:
            after_backward(self)
        self._ev_set[self._cur].record(torch.cuda.current_stream(self.dev))
        self._graph_update()

    def _graph_update(self):
        """the optimiser half of a captured step on the main stream (+ the log row, launched here because g_update is
        shared by both buffer sets while the row reads the step's own set)"""
        self.allreduce()
        if self.g_update is None:
            self.optimizer_step()
        else:
            self._replay(self.g_update[self._gcur])
            if self._n_gbuf == 2:
                self._gcur ^= 1
        self._log_step()

    def train_step(self, sample=True, after_backward=None):
        """one full training step incl. the occupancy refresh cadence of reference train.py:160-163. after_backward(self),
        if given, is called once the step's gradients (self.G) are complete and before the optimiser consumes and
        clears them"""
        if self._log_pending:
            self._log_guard()
        if self.lr_schedule is not None:
            lr = self.lr_schedule.lr_at_step(self.host_step)
            if lr != self.lr:
                self.set_lr(lr)
        refresh = self.host_step % self.update_interval == 0
        if refresh:
            if self._staged is not None:
                torch.cuda.current_stream(self.dev).wait_stream(self._side)  # a staged copy may still be in flight
            self.update_density_grid(warmup=self.host_step < self.warmup_steps)
        if not (self.graph and self._graph_samples == sample):
            self._prepare(sample)
            self._compute()
            if after_backward is not None:
                after_backward(self)
            self._update()
            self._premarched = False
            self.host_step += 1
            return
        main = torch.cuda.current_stream(self.dev)
        if self._staged is not None:  # a host batch staged (copied [+ marched]) by stage_batch()
            self._cur = self._staged
            self._staged = None
            main.wait_stream(self._side)
            if refresh:  # staged ahead of a refresh: march now, against the refreshed grid (the reference's ordering)
                self._replay(self.g_prepare[self._cur])
            self._graph_compute_update(after_backward)
            self._premarched = False
            self._inflight = True
            self.host_step += 1
            return
        if self._premarched:
            self._cur = 1 - self._cur  # the set the previous step marched ahead
        else:
            self._replay(self.g_prepare[self._cur])
        # deep pipeline: the next step's batch + march into the OTHER set (side stream) under this whole step
        ahead = sample and ((self.host_step + 1) % self.update_interval != 0)
        if ahead:
            # the other set's last reader is the previous step's compute: once that is done (and this step's march, if it
            # ran on the main stream, is enqueued) the next march may start -- it does not wait for the optimiser
            if self._premarched:
                self._side.wait_event(self._ev_set[1 - self._cur])
            else:
                self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                self._replay(self.g_prepare[1 - self._cur])
        self._graph_compute_update(after_backward)
        if ahead:
            main.wait_stream(self._side)
        self._premarched = ahead
        self.host_step += 1

    # ---- read-backs (these DO synchronise; not used inside the timed loop) -----------------------------------
    def stats(self):
        c = self.counters.tolist()
        s = self.scalars.tolist()
        n = self.n_rays
        mse = s[2] / (3 * n)
        loss = mse + self.cfg.lambda_opacity * s[3] / n
        out = dict(rm_samples=c[2], vr_samples=c[3], bw_samples=c[5] if self.live_idx is not None else c[2], mse=mse, psnr=-10 * math.log10(max(mse, 1e-12)))
        if self.lambda_distortion > 0:
            out["distortion"] = self.lambda_distortion * float(self.dist_loss.mean())
            loss += out["distortion"]
        out["loss"] = loss
        return out

    # ---- the per-step log (Trainer(log_rows=R)) -------------------------------------------------------------
    def drain_log(self, wait=False):
        """Every step's stats() without synchronising the host. Enqueues one device-to-host copy of the log rows written
        since the last drain (on a side stream, behind an event recorded on the current stream, into pinned memory) and
        returns, in step order, the rows of earlier drains whose copies have completed, as the dicts of
        log_rows_to_stats(): stats()'s keys plus 'step' and 'lr'. wait=True also waits for the copies still in flight
        (for tests and the end of a run). Call it at least every log_rows steps: if more steps have passed, their oldest
        rows are overwritten and it raises (the rows of the earlier drains are kept for the next call)."""
        if self.log_ring is None:
            raise RuntimeError("Trainer.drain_log: the per-step log is off (construct the Trainer with log_rows > 0)")
        R = self.log_rows
        first, n = self._log_next, self.host_step - self._log_next
        if n > R:
            self._log_next = self.host_step
            raise RuntimeError("Trainer.drain_log: %d steps since the last drain, the log ring holds %d: the rows of steps "
                               "%d..%d are overwritten (drain at least every log_rows steps)" % (n, R, first, self.host_step - R - 1))
        if n > 0:
            with torch.cuda.device(self.dev):
                main = torch.cuda.current_stream(self.dev)
                if self._log_stream is None:
                    self._log_stream = torch.cuda.Stream(self.dev)
                    self.log_ring.record_stream(self._log_stream)
                ready = torch.cuda.Event()
                ready.record(main)
                self._log_stream.wait_event(ready)
                host = torch.empty(n, 8, dtype=torch.int32, pin_memory=True)
                at = 0
                with torch.cuda.stream(self._log_stream):
                    for lo, hi in log_ring_spans(first, n, R):
                        host[at:at + hi - lo].copy_(self.log_ring[lo:hi], non_blocking=True)
                        at += hi - lo
                done = torch.cuda.Event()
                done.record(self._log_stream)
            self._log_pending.append((first, n, host, done))
            self._log_next = self.host_step
        out = []
        while self._log_pending:
            first, n, host, done = self._log_pending[0]
            if wait:
                done.synchronize()
            elif not done.query():
                break
            self._log_pending.pop(0)
            rows = log_rows_to_stats(host.numpy(), self.n_rays, self.cfg.lambda_opacity, self.lambda_distortion,
                                     self.live_idx is not None)
            if [r["step"] for r in rows] != list(range(first, first + n)):
                raise RuntimeError("Trainer.drain_log: the log rows are not those of steps %d..%d (was the optimiser "
                                   "stepped outside train_step?)" % (first, first + n - 1))
            out += rows
        return out

    def _log_guard(self):
        """a copy still in flight may hold the row the coming step overwrites: the step waits for that copy"""
        s = self.host_step - self.log_rows
        for first, n, _, done in self._log_pending:
            if first <= s < first + n:
                torch.cuda.current_stream(self.dev).wait_event(done)
