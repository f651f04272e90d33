"""One optimisation step of the reference's training loop as ONE replayed CUDA graph (SURVEY.md 8f rank 2).

`run_nerf.train()` does, per iteration (run_nerf.py:757-784): render the ray batch with `retraw=True`, two `img2mse`
terms, `loss.backward()`, `optimizer.step()` (Adam over 48 tensors), then the exponential learning-rate decay on the
host.  Through the drop-in that is ~40 library launches plus autograd and optimizer bookkeeping in Python; after the
fusion the GPU work is a few milliseconds, so the host side matters.  `FusedTrainStep` runs the same arithmetic with
no autograd graph and no per-tensor optimizer:

    pack weights -> pack rays -> z sampling -> fused pass (coarse, training mode) -> resampling -> fused pass (fine)
    -> fused MSE + gradient seed (both terms) -> tensor-core backward of both passes into ONE flat gradient buffer
    (the fp16 path, or under precision tc_split with set_backward('tc_split') the split one: api._train_path)
    -> [one all-reduce of that buffer when data parallel] -> flat Adam with the decayed rate computed on the device

captured once per ray count and replayed.  The constructor's `n_rays` is the capacity: the buffers hold that many rays and
its graph is captured at once; a step of fewer rays (the short last batch of an epoch) runs on the first rows of the same
buffers under a graph of its own, captured on first use.  The parameters stay the SAME `nn.Parameter` objects (re-pointed at
slices of one flat buffer), so `state_dict()` / checkpoints / `render()` keep working; `attach_optimizer()` exposes the
moments to a `torch.optim.Adam` so that the reference's checkpoint format (run_nerf.py:792-800) is unchanged, and
`load_optimizer()` takes them back from one (run_nerf.py:215-233 reloads it).  `state_dict()` / `load_state_dict()` add what
a bit-exact continuation needs on top, stored under `RESUME_KEY` of the same checkpoint dict (INTEGRATION §5a).
No reference counterpart; nothing here is needed by the drop-in path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import api
from ._lib import NerfPassOut, check

# The key of the reference's checkpoint dict under which a continuation's extra state goes: {"train_step":
# FusedTrainStep.state_dict(), "batcher": DeviceRayBatcher.state_dict()}.  The reference's create_nerf reads only its own four
# keys (run_nerf.py:225-233), so it still reloads such a file.
RESUME_KEY = "nerf_b200_resume"


def adam_moments(named_params, optimizer, betas, eps):
    """The Adam state that `optimizer` holds for `named_params` ((name, Parameter) pairs in the order of the flat buffer), matched
    by parameter identity, not by position in its param_groups.  -> None when it holds state for none of them, else
    (step, [(offset in the flat buffer, exp_avg, exp_avg_sq) per parameter]).  `step` may be a tensor (current torch) or an int
    (torch 1.11, which the reference pins and its published checkpoints were written with).  Raises RuntimeError for a parameter
    the optimizer does not hold, hyper-parameters the flat Adam does not share (betas, eps, weight decay, amsgrad, maximize),
    state for some parameters only, a moment whose shape is not its parameter's, or step counts that differ."""
    named_params = list(named_params)
    group_of = {id(q): g for g in optimizer.param_groups for q in g["params"]}
    offsets, off = [], 0
    for name, p in named_params:
        g = group_of.get(id(p))
        if g is None:
            raise RuntimeError(f"load_optimizer: parameter {name} is not in the optimizer")
        if tuple(float(b) for b in g["betas"]) != tuple(float(b) for b in betas) or float(g["eps"]) != float(eps):
            raise RuntimeError(f"load_optimizer: the optimizer's betas {tuple(g['betas'])} / eps {g['eps']} for {name} differ from the "
                               f"step's own {tuple(betas)} / {eps}")
        if g.get("weight_decay", 0) or g.get("amsgrad", False) or g.get("maximize", False):
            raise RuntimeError(f"load_optimizer: {name} is in a param group with weight_decay, amsgrad or maximize, which the flat Adam "
                               "does not implement")
        offsets.append(off)
        off += p.numel()
    states = [optimizer.state.get(p) for _, p in named_params]
    given = [bool(s) for s in states]
    if not any(given):
        return None
    if not all(given):
        missing = [name for (name, _), h in zip(named_params, given) if not h]
        raise RuntimeError(f"load_optimizer: the optimizer holds Adam state for {sum(given)} of {len(given)} parameters; "
                           f"none for {', '.join(missing[:4])}{' ...' if len(missing) > 4 else ''}")
    steps, out = {}, []
    for (name, p), s, o in zip(named_params, states, offsets):
        for k in ("step", "exp_avg", "exp_avg_sq"):
            if k not in s:
                raise RuntimeError(f"load_optimizer: the optimizer's state for {name} has no '{k}'")
        for k in ("exp_avg", "exp_avg_sq"):
            if tuple(s[k].shape) != tuple(p.shape):
                raise RuntimeError(f"load_optimizer: {k} of {name} has shape {tuple(s[k].shape)}, the parameter {tuple(p.shape)}")
        steps.setdefault(float(s["step"]), name)
        out.append((o, s["exp_avg"], s["exp_avg_sq"]))
    if len(steps) != 1:
        raise RuntimeError("load_optimizer: the parameters' Adam step counts differ: " +
                           ", ".join(f"{t:g} ({name})" for t, name in sorted(steps.items())))
    step = next(iter(steps))
    if step != int(step) or not 0 <= step < 2 ** 24:          # the flat Adam counts steps in a float32
        raise RuntimeError(f"load_optimizer: Adam step count {step} is not a whole number in [0, 2^24)")
    return int(step), out


class FusedTrainStep:
    def __init__(self, H, W, K, n_rays, render_kwargs, lrate=5e-4, lrate_decay=250, betas=(0.9, 0.999), eps=1e-8,
                 process_group=None, use_graph=True, data_parallel=True):
        """render_kwargs: the `render_kwargs_train` dict of create_nerf() plus near / far (run_nerf.py:643-648).
        n_rays: the most rays a step takes (N_rand); the graph of an n_rays step is captured here.
        lrate_decay is in units of 1000 steps like the reference's --lrate_decay (run_nerf.py:779-780)."""
        import torch.distributed as dist
        self.lib = _lib.load()
        kw = dict(render_kwargs)
        self.net_c, self.net_f = kw["network_fn"], kw.get("network_fine")
        if not isinstance(self.net_c, api.NeRF):
            raise RuntimeError("FusedTrainStep needs nerf_b200.NeRF networks (with or without view directions)")
        self.use_viewdirs = bool(self.net_c.use_viewdirs)
        self.Sc, self.Ni = int(kw["N_samples"]), int(kw.get("N_importance", 0))
        if self.Ni > 0 and self.net_f is None:
            self.net_f = self.net_c
        self.path = api._train_path(api.get_precision(), api.get_backward(), True, self.net_c, self.net_f if self.Ni > 0 else None,
                                    fused=True)
        self.dev = self.net_c._check_device()
        self.H, self.W, self.K, self.N = int(H), int(W), K, int(n_rays)
        self.ray_stride = 11 if self.use_viewdirs else 8
        q = kw.get("network_query_fn")
        self.cfgd = dict(N_samples=self.Sc, N_importance=self.Ni, multires=int(getattr(q, "multires", 10)),
                         multires_views=int(getattr(q, "multires_views", 4)), lindisp=bool(kw.get("lindisp", False)),
                         perturb=float(kw.get("perturb", 0.)), white_bkgd=bool(kw.get("white_bkgd", False)), retraw=True)
        self.noise_std = float(kw.get("raw_noise_std", 0.))
        self.ndc, self.near, self.far = int(bool(kw.get("ndc", True))), float(kw.get("near", 0.)), float(kw.get("far", 1.))
        self.lr0, self.decay_rate, self.decay_steps = float(lrate), 0.1, float(lrate_decay) * 1000.0
        self.b1, self.b2, self.eps = float(betas[0]), float(betas[1]), float(eps)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if (data_parallel and dist.is_available() and dist.is_initialized()) else 1
        # ---- one flat buffer for parameters, gradients and moments; the Parameters become views of it ----
        nets = [self.net_c] + ([self.net_f] if (self.net_f is not None and self.net_f is not self.net_c) else [])
        self.params = [p for n in nets for p in n.parameters()]
        total = sum(p.numel() for p in self.params)
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.flat_p = torch.empty(total, **f32)
        self.flat_g = torch.zeros(total, **f32)
        self.m, self.v = torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.state = torch.zeros(4, **f32)          # [0] loss of the last step, [1] steps taken, [2] rate of the last step
        off, self._gviews = 0, {}
        with torch.no_grad():
            for p in self.params:
                n = p.numel()
                self.flat_p[off:off + n].copy_(p.reshape(-1))
                p.data = self.flat_p[off:off + n].view_as(p)
                p.grad = self.flat_g[off:off + n].view_as(p)
                off += n
        self._gs = []
        for n in nets:
            self._gs.append(n.grad_struct({k: p.grad for k, p in n.named_parameters()}))
        self._nets = nets
        # ---- fixed buffers of the step ----
        N, Sc, Sf = self.N, self.Sc, self.Sc + self.Ni
        self.rays = torch.zeros((2, N, 3), **f32)
        self.rays[1, :, 2] = -1.0
        self.target = torch.zeros((N, 3), **f32)
        self.packed_rays = torch.empty((N, self.ray_stride), **f32)
        self.t_rand = torch.zeros((N, Sc), **f32) if self.cfgd["perturb"] > 0 else None
        self.u_rand = torch.zeros((N, self.Ni), **f32) if (self.cfgd["perturb"] > 0 and self.Ni > 0) else None
        self.noise0 = torch.zeros((N, Sc), **f32) if self.noise_std > 0 else None
        self.noise1 = torch.zeros((N, Sf), **f32) if (self.noise_std > 0 and self.Ni > 0) else None
        self.t_vals = torch.linspace(0., 1., steps=Sc, device=self.dev)
        self.u_det = torch.linspace(0., 1., steps=self.Ni, device=self.dev) if self.Ni > 0 else None
        self.z_c, self.z_f, self.z_std = torch.empty((N, Sc), **f32), torch.empty((N, max(Sf, 1)), **f32), torch.empty((N,), **f32)
        o = {k: torch.empty(s, **f32) for k, s in (("rgb0", (N, 3)), ("disp0", (N,)), ("acc0", (N,)), ("w0", (N, Sc)), ("raw0", (N, Sc, 4)),
                                                   ("rgb", (N, 3)), ("disp", (N,)), ("acc", (N,)), ("raw", (N, Sf, 4)),
                                                   ("g_rgb", (N, 3)), ("g_rgb0", (N, 3)))}
        self.out = o
        self._out_c = NerfPassOut(api._ptr(o["rgb0"]), api._ptr(o["disp0"]), api._ptr(o["acc0"]), C.c_void_p(0), api._ptr(o["w0"]), api._ptr(o["raw0"]))
        self._out_f = NerfPassOut(api._ptr(o["rgb"]), api._ptr(o["disp"]), api._ptr(o["acc"]), C.c_void_p(0), C.c_void_p(0), api._ptr(o["raw"]))
        self._np_c, self._np_f = self.net_c.net_params(), (self.net_f.net_params() if self.Ni > 0 else None)
        lib = self.lib
        self._pack_fn = getattr(lib, self.path.pack_weights)
        packed_bytes = getattr(lib, self.path.packed_bytes)
        self._pk_c = torch.empty(packed_bytes(C.byref(self._np_c)), dtype=torch.uint8, device=self.dev)
        self._pk_f = self._pk_c if (self.Ni == 0 or self.net_f is self.net_c) else \
            torch.empty(packed_bytes(C.byref(self._np_f)), dtype=torch.uint8, device=self.dev)
        # the seeds of a path without an rgb-only backward (split): NerfOutGrads of dL/drgb_map of each pass
        self._og_c = _lib.NerfOutGrads(rgb_map=api._ptr(o["g_rgb0"]))
        self._og_f = _lib.NerfOutGrads(rgb_map=api._ptr(o["g_rgb"]))
        # every buffer above has the rays as its leading dimension, so an n-ray step (n <= N) runs on their first n rows, which
        # start at the same pointers; the records and workspaces follow the tile plan of n (see _size_buffers)
        self._sized = {}
        self._sized[N] = self._size_buffers(N)
        self._cam = api._camera(self.H, self.W, self.K)
        self._cfg = api._cfg_struct(self.cfgd, self.ray_stride)
        self.host_loss = torch.zeros(4, dtype=torch.float32, device="cpu").pin_memory()
        # ---- capture ----
        self.graph = self.graph_adam = None
        self._graphs = {}                               # n -> the graph of an n-ray step; other sizes are captured on first use
        if use_graph:
            self.graph = self._graphs[N] = self._capture(N)
            if self.world > 1:
                self.graph_adam = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_adam):
                    self._adam()

    def _size_buffers(self, n):
        """The training records, the workspaces and the backward-pass descriptors of an n-ray step.  Their sizes follow the
        tile plan the library derives from n, which can need more for some n < N than for N, so each is the capacity's
        where the library's size query for n fits in it, and a new buffer of the queried size otherwise."""
        lib, dev, fine, Sf = self.lib, self.dev, self.Ni > 0, self.Sc + self.Ni
        cap = self._sized.get(self.N)

        def buf(key, nbytes):
            t = None if cap is None else cap[key]
            return t if (t is not None and t.numel() >= nbytes) else torch.empty(nbytes, dtype=torch.uint8, device=dev)
        b = {}
        with api._on(self.rays):
            for tag, S, np_ in (("c", self.Sc, self._np_c), ("f", Sf, self._np_f))[:1 + fine]:
                ab, mb = api._record_bytes(lib, self.path, n, S, np_)
                b["act_" + tag], b["mask_" + tag] = buf("act_" + tag, ab), buf("mask_" + tag, mb)
            b["ws"] = buf("ws", lib.nerf_b200_march_workspace_bytes(n, Sf))
            bw = getattr(lib, self.path.bwd_ws)(n, self.Sc, C.byref(self._np_c), Sf if fine else 0, C.byref(self._np_f) if fine else None)
            b["bws"] = buf("bws", bw + 1024)
        if cap is not None and all(b[k] is cap[k] for k in b):
            return cap
        o = self.out
        b["sv_c"] = api._records_save(b["act_c"], b["mask_c"])
        b["bp_c"] = api._bwd_pass(self.z_c, self.noise0, self.Sc, self._np_c, self._pk_c, o["raw0"], b["sv_c"], o["g_rgb0"], self._gs[0])
        b["sv_f"] = b["bp_f"] = None
        if fine:
            b["sv_f"] = api._records_save(b["act_f"], b["mask_f"])
            b["bp_f"] = api._bwd_pass(self.z_f, self.noise1, Sf, self._np_f, self._pk_f, o["raw"], b["sv_f"], o["g_rgb"], self._gs[-1])
        return b

    def _capture(self, n, pool=None, keep_rng=False):
        """The CUDA graph of an n-ray step: everything after the ray packing (before Adam when data parallel), captured after
        two eager warm-up steps whose changes to the parameters, moments and state are undone."""
        snap = (self.flat_p.clone(), self.m.clone(), self.v.clone(), self.state.clone())

        def warm_up():                                  # opt-ins, caches, lazy initialisations outside the capture
            for _ in range(2):
                self._pack_rays(n=n); self._fwd_bwd(n); self._adam()

        def body():
            self._fwd_bwd(n)
            if self.world == 1:
                self._adam()
        graph, _ = api._capture_graph(self.dev, warm_up, body, pool=pool, keep_rng=keep_rng)
        with torch.no_grad():                           # the warm-up steps must not count: restore parameters and moments
            self.flat_p.copy_(snap[0]); self.m.copy_(snap[1]); self.v.copy_(snap[2]); self.state.copy_(snap[3])
        return graph

    # ---- the step, as library calls on the current stream; n rays (default: the capacity N) ----
    def _pack_rays(self, c2w=None, pixel_index=None, n=None):
        """The ray batch -> packed [n,11] rows ([n,8] without view directions).  Outside the graph (one launch): the camera travels
        in the kernel arguments, so a per-step pose could not be replayed.  Given rays (self.rays) or -- SURVEY 8f rank 3 -- pixels of
        one posed image."""
        n = self.N if n is None else n
        vd = int(self.use_viewdirs)
        with api._on(self.rays):
            if pixel_index is None:
                check(self.lib.nerf_b200_pack_rays(api._ptr(self.rays[0]), api._ptr(self.rays[1]), None, C.byref(self._cam), n, 0, self.ndc, self.near,
                                                   self.far, vd, api._ptr(self.packed_rays), api._stream(self.rays)), "pack_rays")
            else:
                cam = api._camera(self.H, self.W, self.K, c2w)
                check(self.lib.nerf_b200_pack_rays_pixels(C.byref(cam), api._ptr(pixel_index), n, self.ndc, self.near, self.far, vd,
                                                          api._ptr(self.packed_rays), api._stream(self.rays)), "pack_rays_pixels")

    def _fwd_bwd(self, n=None):
        lib, cfg = self.lib, self._cfg
        n = self.N if n is None else n
        b = self._sized[n]
        st = api._stream(self.rays)
        with api._on(self.rays):
            check(self._pack_fn(C.byref(self._np_c), api._ptr(self._pk_c), self._pk_c.numel(), st), "pack_weights")
            if self._pk_f is not self._pk_c:
                check(self._pack_fn(C.byref(self._np_f), api._ptr(self._pk_f), self._pk_f.numel(), st), "pack_weights")
            # the draws of an n-ray step fill the first n rows only: the generator advances as in a step built for n rays
            if self.t_rand is not None:                                 # (the reference's draw order)
                self.t_rand[:n].uniform_()                              # run_nerf.py:371
            if self.noise0 is not None:
                self.noise0[:n].normal_().mul_(self.noise_std)          # run_nerf.py:285
            if self.u_rand is not None:
                self.u_rand[:n].uniform_()                              # run_nerf_helpers.py:208
            if self.noise1 is not None:
                self.noise1[:n].normal_().mul_(self.noise_std)
            fine = self.Ni > 0
            api._call(lib, self.path.fwd, api._ptr(self.packed_rays), n, C.byref(cfg), C.byref(self._np_c), api._ptr(self._pk_c),
                      C.byref(self._np_f) if fine else None, api._ptr(self._pk_f) if fine else None,
                      api._ptr(self.t_vals), api._ptr(self.u_det), api._ptr(self.t_rand), api._ptr(self.u_rand), api._ptr(self.noise0),
                      api._ptr(self.noise1), api._ptr(self.z_c), C.byref(self._out_c), api._ptr(self.z_f) if fine else None,
                      api._ptr(self.z_std) if fine else None, C.byref(self._out_f) if fine else None, api._ptr(b["ws"]), b["ws"].numel(),
                      C.byref(b["sv_c"]), C.byref(b["sv_f"]) if fine else None, st)
            # loss = img2mse(rgb, target) + img2mse(rgb0, target)  (run_nerf.py:764-772), means over the n rays, and its gradient seeds
            self.state[0:1].zero_()
            self.flat_g.zero_()
            gscale = 1.0 / self.world
            o = self.out
            if fine:
                check(lib.nerf_b200_mse_seed(api._ptr(o["rgb"]), api._ptr(self.target), n, gscale, api._ptr(o["g_rgb"]), api._ptr(self.state), st), "mse_seed")
            check(lib.nerf_b200_mse_seed(api._ptr(o["rgb0"]), api._ptr(self.target), n, gscale, api._ptr(o["g_rgb0"]), api._ptr(self.state), st), "mse_seed")
            # backward of both passes into the flat gradient buffer (one call): the seeds in NerfBwdPass.g_rgb where the path has an
            # rgb-only backward, else as NerfOutGrads
            seeds = () if self.path.bwd_rgb else (C.byref(self._og_c), C.byref(self._og_f) if fine else None)
            api._call(lib, self.path.bwd_rgb or self.path.bwd, api._ptr(self.packed_rays), n, C.byref(cfg), C.byref(b["bp_c"]),
                      C.byref(b["bp_f"]) if fine else None, *seeds, api._ptr(b["bws"]), b["bws"].numel(), st)

    def _adam(self):
        with api._on(self.rays):
            check(self.lib.nerf_b200_adam_step(api._ptr(self.flat_p), api._ptr(self.flat_g), api._ptr(self.m), api._ptr(self.v), self.flat_p.numel(),
                                               api._ptr(self.state), self.lr0, self.decay_rate, self.decay_steps, self.b1, self.b2, self.eps, 1.0,
                                               api._stream(self.rays)), "adam_step")

    def _prepare(self, n):
        """The buffers of an n-ray step and, with graphs, its graph: made on the first step of that size.  A new size is
        captured in the first graph's memory pool (the graphs never run concurrently), and the capture's warm-up leaves the
        device's generator where it was, so the step draws what it would have drawn without the capture."""
        if n not in self._sized:
            self._sized[n] = self._size_buffers(n)
        if self.graph is not None and n not in self._graphs:
            self._graphs[n] = self._capture(n, pool=self.graph.pool(), keep_rng=True)
        return self._graphs.get(n)

    def _check_size(self, n):
        if not 0 < n <= self.N:
            raise RuntimeError(f"FusedTrainStep: a step of {n} rays; this step takes 1 to {self.N} (its n_rays)")
        return n

    # ---- public ----
    def step_device(self, c2w=None, pixel_index=None, n_rays=None):
        """One step on the first n rows of the rays / target already in `self.rays` ([2,N,3]) and `self.target` ([N,3]); no
        host sync.  With `c2w` [3,4] and `pixel_index` (int64 CUDA tensor [n] of row-major pixel ids) the rays are generated on
        the device for those pixels of that pose instead (run_nerf.py:728-757 without get_rays' [H,W,3] tensors).
        n is `n_rays`, else `pixel_index.numel()`, else the capacity N; 0 < n <= N.  The loss is the mean over the n rays, as
        img2mse takes it, and the random draws are those of a step built for n rays.  The first step of a size other than N
        captures its graph (see _prepare)."""
        import torch.distributed as dist
        n = self._check_size(int(n_rays) if n_rays is not None else (pixel_index.numel() if pixel_index is not None else self.N))
        if pixel_index is not None and pixel_index.numel() != n:
            raise RuntimeError(f"FusedTrainStep: pixel_index has {pixel_index.numel()} entries for a step of {n} rays")
        graph = self._prepare(n)                        # before the packing: a capture's warm-up packs self.rays
        self._pack_rays(c2w, pixel_index, n)
        if graph is not None:
            graph.replay()
        else:
            self._fwd_bwd(n)
        if self.world > 1:
            dist.all_reduce(self.flat_g, op=dist.ReduceOp.SUM, group=self.group)     # ONE collective: every gradient, 4.77 MB
            if self.graph_adam is not None:
                self.graph_adam.replay()
            else:
                self._adam()
        elif self.graph is None:
            self._adam()
        for n in self._nets:
            n.invalidate_pack()                         # parameters changed behind autograd's version counters

    def __call__(self, rays_host, target_host):
        """rays_host [2,n,3], target_host [n,3] with 0 < n <= N (pinned host memory makes the copies asynchronous) -> loss
        (python float).  Copies the batch into the first n rows, runs the step, copies the loss out and synchronises the stream."""
        sr, st = tuple(rays_host.shape), tuple(target_host.shape)
        if len(sr) != 3 or sr[0] != 2 or sr[2] != 3 or st != (sr[1], 3):
            raise RuntimeError(f"FusedTrainStep: rays {sr} and target {st}; expected [2, n, 3] and [n, 3]")
        n = self._check_size(sr[1])
        self.rays[:, :n].copy_(rays_host, non_blocking=True)
        self.target[:n].copy_(target_host, non_blocking=True)
        self.step_device(n_rays=n)
        self.host_loss.copy_(self.state, non_blocking=True)
        torch.cuda.current_stream(self.dev).synchronize()
        return float(self.host_loss[0])

    @property
    def global_step(self) -> int:
        return int(self.state[1].item())

    def attach_optimizer(self, optimizer: torch.optim.Adam):
        """Make `optimizer`'s per-parameter state alias this step's flat moments, so optimizer.state_dict() (the
        reference's checkpoint content, run_nerf.py:796-799) reflects the fused steps."""
        off = 0
        step = self.state[1].detach().clone().cpu()
        for p in self.params:
            n = p.numel()
            optimizer.state[p] = {"step": step.clone(), "exp_avg": self.m[off:off + n].view_as(p), "exp_avg_sq": self.v[off:off + n].view_as(p)}
            off += n
        t = float(self.state[1].item())
        for g in optimizer.param_groups:                # the rate the NEXT step will use, as run_nerf.py:779-783 leaves it
            g["lr"] = self.lr0 * self.decay_rate ** ((t - 1.0) / self.decay_steps) if (t >= 1.0 and self.decay_steps > 0) else self.lr0
        return optimizer

    def _named_params(self):
        return [(f"{tag}.{k}", p) for tag, n in zip(("network_fn", "network_fine"), self._nets) for k, p in n.named_parameters()]

    def load_optimizer(self, optimizer: torch.optim.Adam):
        """The inverse of attach_optimizer: continue from the Adam state `optimizer` holds, e.g. after create_nerf() reloaded a
        checkpoint (run_nerf.py:225-228).  Each parameter's exp_avg / exp_avg_sq is found by parameter identity and copied into
        the flat moments, and the step count goes to state[1], from which the device derives the decayed rate and the bias
        correction.  The count is Adam's `step`, the number of updates applied; the checkpoint's `global_step` is not read (the
        reference writes it before its increment, run_nerf.py:794 / :872, so in its own checkpoints it is one less).  An
        optimizer without state (a fresh run) leaves the step as it is.  Afterwards the optimizer's state aliases the flat
        moments, as after attach_optimizer.  The learning rate comes from the step's own lrate / lrate_decay, not from the
        optimizer's param_groups.  See adam_moments for what is refused."""
        found = adam_moments(self._named_params(), optimizer, (self.b1, self.b2), self.eps)
        if found is not None:
            step, moments = found
            with torch.no_grad():
                for off, m, v in moments:
                    self.m[off:off + m.numel()].copy_(m.reshape(-1))
                    self.v[off:off + v.numel()].copy_(v.reshape(-1))
                self.state[1] = float(step)
        return self.attach_optimizer(optimizer)

    def state_dict(self):
        """What a bit-exact continuation needs besides the networks and the optimizer: the flat moments, the step state (loss,
        step count, rate) and the state of this device's CUDA generator, from which the step's draws (t_rand, σ noise, u) and
        DeviceRayBatcher's device draws come.  m / v / state are this step's own buffers, as nn.Module.state_dict returns the
        parameters themselves, so torch.save stores them once together with the optimizer state that attach_optimizer aliased
        to them."""
        return {"m": self.m, "v": self.v, "state": self.state, "cuda_rng_state": torch.cuda.get_rng_state(self.dev)}

    def load_state_dict(self, sd):
        """The inverse of state_dict().  Call it after construction: the constructor's warm-up steps draw from the generator.
        The captured graph reads the generator's seed and offset at every replay, so its replays then draw what the
        interrupted run would have drawn.  In a data-parallel run every rank loads the same dict (INTEGRATION §5a)."""
        with torch.no_grad():
            for k, dst in (("m", self.m), ("v", self.v), ("state", self.state)):
                if tuple(sd[k].shape) != tuple(dst.shape):
                    raise RuntimeError(f"FusedTrainStep.load_state_dict: '{k}' has shape {tuple(sd[k].shape)}, this step's {tuple(dst.shape)}")
                dst.copy_(sd[k])
        torch.cuda.set_rng_state(sd["cuda_rng_state"].cpu(), self.dev)
