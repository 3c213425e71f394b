"""Policy optimisation with batched random restarts (replaces the sequential restart loop of
``PILCO.optimize_policy``, pilco/models/pilco.py:75-113).

* All restarts of this rank are evaluated in ONE batched device rollout (forward + reverse sweep).
* Each restart is driven by its own SciPy L-BFGS-B instance (the optimiser the reference uses through
  ``gpflow.optimizers.Scipy``); the instances run in worker threads that advance in lock step, so every
  device call evaluates the current trial points of all still-active restarts.
* The restarts of a rank are independent optimisation problems, so they are dealt to ``GROUPS`` lock-step groups
  that only wait for THEIR OWN previous evaluation: each group has its own evaluator (captured graph, stream, pinned
  buffers) and driver thread, started half an evaluation apart, so the latency-bound reverse sweep and the SciPy
  host work of one group run under the tile kernels of the other.
* Multi-GPU: restart r belongs to rank r % world; after the local optimisations a single
  ``all_gather`` of ``[loss | flat parameters]`` lets every rank pick the same winner (ties -> lowest
  restart index, the sequential ``>`` comparison of pilco.py:105).  No other collective is used.
"""
import os
import threading
import time

import numpy as np
import scipy.optimize
import torch

from . import engine, controllers, _lib

BIG = 1e10
LAST_STATS = {}          # filled by optimize(): evaluator calls, restarts on this rank, horizon (bench.py reads it)
GROUPS = 2               # lock-step groups per rank (env PILCO_OPT_GROUPS); a group keeps at least MIN_GROUP restarts
MIN_GROUP = 8


def group_bounds(R, groups=None):
    """[lo, hi) slices of the R local restarts dealt to the lock-step groups."""
    g = int(os.environ.get("PILCO_OPT_GROUPS", GROUPS) if groups is None else groups)
    g = max(1, min(g, R // MIN_GROUP if R >= MIN_GROUP else 1))
    b = [round(k * R / g) for k in range(g + 1)]
    return [(b[k], b[k + 1]) for k in range(g)]


class _FlatEvaluator:
    """What the evaluators share: loss and gradient for R flat policy parameter vectors (``controller.get_flat()``
    layout), served through pinned host buffers, on the evaluator's own stream, with the whole evaluation captured in
    one CUDA graph.  A subclass builds its plans, then calls ``_setup_io()``, and implements ``_enqueue()`` with
    ``_unpack`` (flat parameters -> policy buffers) and ``_pack`` (loss, status and gradient -> ``d_out``)."""

    def __init__(self, pilco, R):
        self.pilco, self.R = pilco, R
        c = pilco.controller
        self.c = c
        self.sched = isinstance(c, controllers.TimeVaryingLinearController)     # per-step W_t, b_t
        self.linear = isinstance(c, controllers.LinearController) or self.sched
        self.mlp = isinstance(c, controllers.MlpController)                      # theta as the flat vector itself
        self.flat0 = np.tile(c.get_flat(), (R, 1))
        self.P = self.flat0.shape[1]
        if self.mlp:
            U, Ds = c.control_dim, c.state_dim
        elif self.linear:
            U, Ds = c.W.shape[-2:]
        else:
            bf, Ds, U = c.policy_shapes
            self.ell_lower = float(c.models[0].kernel.lengthscales.transform.lower)
        self.shape = (Ds, U)

    def _setup_io(self):
        R = self.R
        self.stream = torch.cuda.Stream()                      # the group's own stream: evaluations of different
        self.done = torch.cuda.Event()                         # groups overlap on the device
        self.graph, self.ncalls, self.cache, self.eval_s = None, 0, None, 0.0
        self.h_flat = torch.empty((R, self.P), dtype=torch.float64).pin_memory()
        self.h_out = torch.empty((R, self.P + 2), dtype=torch.float64).pin_memory()
        self.d_flat = torch.empty((R, self.P), dtype=torch.float64, device=engine.device())
        self.d_out = torch.empty((R, self.P + 2), dtype=torch.float64, device=engine.device())

    def __call__(self, flats):
        """flats [R,P] (numpy) -> loss [R], grad [R,P]; non-finite restarts get (BIG, 0).
        The first call runs eagerly (warm-up), the second captures the whole evaluation -- parameter unpacking,
        policy factorisation, forward, reverse sweep, gradient packing -- into one CUDA graph that every later
        L-BFGS evaluation replays."""
        flats = np.asarray(flats, dtype=np.float64)
        if self.cache is not None and np.array_equal(flats, self.cache[0]):     # the point prepare() evaluated
            return self.cache[1].copy(), self.cache[2].copy()
        self.h_flat.copy_(torch.as_tensor(flats))
        self.ncalls += 1
        torch.cuda.set_device(self.stream.device)              # (driver threads start on device 0)
        with torch.cuda.stream(self.stream):
            if self.graph is not None:
                self.graph.replay()
            elif self.ncalls == 2 and self.use_graph:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._enqueue()
                self.graph = g
                g.replay()
            else:
                self._enqueue()
            self.done.record()
        self.done.synchronize()
        res = self.h_out.numpy()
        loss, bad, grad = res[:, 0].copy(), res[:, 1] != 0, res[:, 2:].copy()
        bad |= ~np.isfinite(loss) | ~np.isfinite(grad).all(axis=1)
        loss[bad] = BIG
        grad[bad] = 0.0
        return loss, grad

    use_graph = True

    def prepare(self, flats):
        """Warm-up (eager), graph capture and one timed replay at the starting points, on the calling thread (stream
        capture must not run beside another group's evaluations); the result is kept for the optimisers' first call."""
        self.cache = None
        self(flats)
        self(flats)
        t0 = time.perf_counter()
        loss, grad = self(flats)
        self.eval_s = time.perf_counter() - t0
        self.cache = (np.array(flats, dtype=np.float64), loss, grad)

    def _unpack(self, flat, plan, gp):
        """flat [R,P] device rows -> the plan's linear policy buffers, or the RBF policy ``gp`` (refactorised);
        returns the lengthscales' unconstrained theta [R,U,Ds] (RBF) or None"""
        R = flat.shape[0]
        Ds, U = self.shape
        if self.mlp:
            plan.theta.copy_(flat.reshape(plan.theta.shape))
            return None
        if self.sched:                                         # W stays the spec's zeros without feedback
            nW = self.c.horizon * U * Ds if self.c.feedback else 0
            if nW:
                plan.W.copy_(flat[:, :nW].reshape(plan.W.shape))
            plan.b.copy_(flat[:, nW:].reshape(plan.b.shape))
            return None
        if self.linear:
            plan.W.copy_(flat[:, :U * Ds].reshape(plan.W.shape))
            plan.b.copy_(flat[:, U * Ds:].reshape(plan.b.shape))
            return None
        bf = gp.n
        th = flat[:, bf * Ds + bf * U:].reshape(R, U, Ds)
        gp.X.copy_(flat[:, :bf * Ds].reshape(R, bf, Ds))
        gp.Y.copy_(flat[:, bf * Ds:bf * Ds + bf * U].reshape(R, bf, U))
        # ell = lower + log(1 + e^theta): the controller's own transform (controllers.py:100), same formula as
        # params.Softplus.forward on the host (np.logaddexp)
        gp.ell.copy_(self.ell_lower + torch.logaddexp(th, torch.zeros_like(th)))
        engine.gp_refactorize(gp)
        return th

    def _particle_plan(self, P, consistent, exploration, resample, num_features, measurement_noise=None):
        """self.plan, the batched pathwise-gradient plan of the R restarts over P particles (``ConsistentGradPlan``
        with ``consistent``, else ``ParticlePlan``), and self.gp, the RBF policy it refactorises (None otherwise)"""
        pilco, c, flat0 = self.pilco, self.c, self.flat0
        terms, mult_mu = pilco.reward_spec()
        spec = c.policy_spec(flat0) if self.linear or self.mlp else pilco.policy_spec(flat0)
        self.gp = None if self.linear or self.mlp else spec["gp"]
        if consistent:
            self.plan = engine.ConsistentGradPlan(pilco.mgpr.device_gp(), spec, terms, P, int(pilco.horizon),
                                                  mult_mu=mult_mu, R=self.R, exploration=exploration,
                                                  measurement_noise=measurement_noise, schedule=self.sched,
                                                  num_features=num_features)
        else:
            self.plan = engine.ParticlePlan(pilco.mgpr.device_gp(), spec, terms, P, int(pilco.horizon),
                                            mult_mu=mult_mu, grad=True, R=self.R, exploration=exploration,
                                            measurement_noise=measurement_noise, resample=resample,
                                            schedule=self.sched, num_features=num_features)

    def _pack(self, out, value, info, g, th):
        """out [R,P+2] = [-value | status | -gradient in the flat layout]; the lengthscale block goes through the
        softplus: d ell / d theta = sigmoid(theta)"""
        R = out.shape[0]
        Ds, U = self.shape
        out[:, 0] = -value
        out[:, 1] = info.to(torch.float64)
        if self.mlp:
            out[:, 2:] = -g["theta"].reshape(R, -1)
        elif self.sched:                                         # steps 0 .. H-1 of the horizon's: the rest get 0
            nW = self.c.horizon * U * Ds if self.c.feedback else 0
            out[:, 2:] = 0.0
            if nW:
                gW = g["W"].reshape(R, -1)
                out[:, 2:2 + gW.shape[1]] = -gW
            gb = g["b"].reshape(R, -1)
            out[:, 2 + nW:2 + nW + gb.shape[1]] = -gb
        elif self.linear:
            out[:, 2:2 + U * Ds] = -g["W"].reshape(R, -1)
            out[:, 2 + U * Ds:] = -g["b"].reshape(R, -1)
        else:
            bf = g["X"].shape[-2]
            out[:, 2:2 + bf * Ds] = -g["X"].reshape(R, -1)
            out[:, 2 + bf * Ds:2 + bf * Ds + bf * U] = -g["Y"].reshape(R, -1)
            out[:, 2 + bf * Ds + bf * U:] = -(g["ell"].reshape(R, U, Ds) * torch.sigmoid(th)).reshape(R, -1)


class PolicyEvaluator(_FlatEvaluator):
    """loss(flat) = -sum_t E[r(x_t)] (with the PILCO's exploration b != 0: -sum_t (E[r_t] + b sigma_t)) and its
    gradient for a batch of flat policy parameter vectors.

    The R restarts are dealt to ``nsplit`` sub-batches, each with its own RolloutPlan (taped forward + reverse sweep)
    on its own stream inside ONE captured CUDA graph: the latency-bound glue kernels of one sub-batch overlap the tile
    kernels of the others."""

    NSPLIT = 4

    def __init__(self, pilco, R, nsplit=None, m0=None, S0=None):
        """``m0``, ``S0``: the initial state distribution (default pilco.m_init, pilco.S_init)"""
        super().__init__(pilco, R)
        c, flat0 = self.c, self.flat0
        terms, mult_mu = pilco.reward_spec()
        nsplit = max(1, min(int(self.NSPLIT if nsplit is None else nsplit), R // 4 if R >= 8 else 1))
        bounds = [round(k * R / nsplit) for k in range(nsplit + 1)]
        self.slices = [(bounds[k], bounds[k + 1]) for k in range(nsplit) if bounds[k + 1] > bounds[k]]
        self.plans, self.gps = [], []
        dyn = pilco.mgpr.device_gp()
        b = float(getattr(pilco, "exploration", 0.0))
        exploration = b if b != 0.0 else None                  # b = 0: the plans without exploration
        noise = pilco._noise_var() if hasattr(pilco, "_noise_var") else None
        m0 = pilco.m_init if m0 is None else m0
        S0 = pilco.S_init if S0 is None else S0
        for lo, hi in self.slices:
            spec = c.policy_spec(flat0[lo:hi]) if self.linear else pilco.policy_spec(flat0[lo:hi])
            self.gps.append(None if self.linear else spec["gp"])
            self.plans.append(engine.RolloutPlan(dyn, spec, terms, np.asarray(m0, dtype=np.float64).reshape(-1),
                                                 np.asarray(S0, dtype=np.float64), int(pilco.horizon), R=hi - lo,
                                                 mult_mu=mult_mu, grad=True,
                                                 angles=getattr(pilco, "angle_dims", None), exploration=exploration,
                                                 measurement_noise=noise, schedule=self.sched))
        self.side = [torch.cuda.Stream() for _ in self.plans[1:]]
        self._setup_io()

    def _enqueue(self):
        self.d_flat.copy_(self.h_flat, non_blocking=True)
        cur = torch.cuda.current_stream()
        for st in self.side:                                   # fork: sub-batch k >= 1 on its own stream
            st.wait_stream(cur)
        self._enqueue_slice(0)
        for k, st in enumerate(self.side, start=1):
            with torch.cuda.stream(st):
                self._enqueue_slice(k)
        for st in self.side:                                   # join
            cur.wait_stream(st)
        self.h_out.copy_(self.d_out, non_blocking=True)

    def _enqueue_slice(self, k):
        (lo, hi), plan, gp = self.slices[k], self.plans[k], self.gps[k]
        th = self._unpack(self.d_flat[lo:hi], plan, gp)
        plan.forward()
        g = plan.backward()
        self._pack(self.d_out[lo:hi], plan.reward, torch.maximum(plan.info, gp.info if not self.linear else plan.info),
                   g, th)


class ParticleEvaluator(_FlatEvaluator):
    """loss(flat) = -(mean return of P particles) and its pathwise gradient for a batch of flat policy parameter
    vectors, in ``PolicyEvaluator``'s contract.

    The R policies run over the same particles ``x0`` [P,Ds] and standard normals ``eps`` [P,H,Ds] (H = the horizon),
    held fixed, so the objective is a deterministic function of the parameters: one batched device call
    (pilco_particles_rollout_batch_grad) evaluates every restart.  ``consistent=True``: each particle follows one
    function drawn from the dynamics posterior (pilco_particles_rollout_consistent_grad through
    ``engine.ConsistentGradPlan``).  Box terms carry no pathwise gradient, so a reward with them is rejected.
    ``exploration``: a float b makes the objective PILCO's exploration objective over the particles, mean return +
    b sum_t sigma_t with sigma_t the sample spread of step t's reward (pilco_particles_explore_*, DESIGN.md section 24);
    None (the default) is the mean return.  ``resample=True``: Deep PILCO's Gaussian refit at every step
    (pilco_particles_resampled_grad_rollout, DESIGN.md section 26) with the redraw's standard normals ``xi`` [P,H,Ds],
    held fixed like eps.  A ``TimeVaryingLinearController`` runs the scheduled calls (pilco_particles_scheduled_*,
    DESIGN.md section 28), its gradient per step; an ``MlpController`` the MLP calls (pilco_particles_mlp_*, section 29),
    its flat vector being the device's theta.  ``features``: ``engine.feature_draws`` of the P particles, with
    ``consistent=True``: the functions are those random-feature draws (pilco_particles_features_grad_rollout, DESIGN.md
    section 30) and eps is not read (None)."""

    def __init__(self, pilco, R, x0, eps, consistent=False, exploration=None, resample=False, xi=None, features=None):
        _no_box(pilco)
        super().__init__(pilco, R)
        x0 = engine.dev(x0)
        self._particle_plan(int(x0.shape[0]), consistent, exploration, resample,
                            None if features is None else features.F)
        self.plan.set_inputs(x0, eps, xi=xi, features=features)
        self._setup_io()

    def _enqueue(self):
        self.d_flat.copy_(self.h_flat, non_blocking=True)
        th = self._unpack(self.d_flat, self.plan, self.gp)
        g = self.plan.launch_grad()
        info = self.gp.info if self.gp is not None else torch.zeros_like(g["value"])
        self._pack(self.d_out, g["value"].reshape(self.R), info.reshape(self.R), g, th)
        self.h_out.copy_(self.d_out, non_blocking=True)


class StochasticEvaluator(_FlatEvaluator):
    """One lock-step group of R restarts trained by Adam on particles drawn afresh at every iteration (DESIGN.md
    section 32): the objective is the expected return itself, not one fixed sample of it (Deep PILCO, PIPPS).

    The plan is the one ``ParticleEvaluator`` builds for the same arguments (``consistent``, ``exploration``,
    ``resample``, ``num_features``; also ``measurement_noise``).  ``iteration()`` enqueues, on the current stream and
    without host synchronisation:
      1. the draws, each with ``engine.normals`` into a persistent buffer at the counter ``adam.iter``, under its stream
         id: 0 eps0 [P,Ds] (then x0 = m0 + eps0 F', F = the factor of S0 the class's particle methods use), 1 eps
         [P,H,Ds] (not with features), 2 nu (with measurement noise), 3 xi (with ``resample``), 4, 5, 6 zeta, w, eps_y
         and the feature draws (with ``num_features``);
      2. ``_unpack`` of the device parameters ``theta`` [R,n], the plan's ``launch_grad``, ``_pack`` into ``packed``
         [R,n+2];
      3. ``adam.step(theta, packed)``, which advances the counter.
    ``capture()`` runs one eager iteration (warm-up), restores the start and records one iteration as a CUDA graph that
    ``replay()`` runs.  ``held_out()`` returns each restart's value at the current theta on the held-out sample, the
    same draws under stream ids 16 + j at iteration 0."""

    HELD_OUT = 16

    def __init__(self, pilco, R, flats0, num_samples, seed, m0, F0, consistent=False, exploration=None, resample=False,
                 num_features=None, measurement_noise=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, max_norm=None,
                 trace_rows=0):
        _no_box(pilco)
        engine.adam_hyperparameters(lr, betas, eps, max_norm)
        super().__init__(pilco, R)
        P, self.seed = int(num_samples), int(seed)
        self._particle_plan(P, consistent, exploration, resample, num_features, measurement_noise)
        p, d = self.plan, engine.device()
        mk = lambda *shape: torch.zeros(shape, dtype=torch.float64, device=d)
        self.flats0 = engine.dev(np.asarray(flats0, dtype=np.float64).reshape(R, self.P))
        self.theta, self.packed = self.flats0.clone(), mk(R, self.P + 2)
        self.adam = engine.AdamState(R, self.P, lr, betas, eps, max_norm, trace_rows)
        self.zero = torch.zeros(1, dtype=torch.int64, device=d)            # the held-out sample's iteration
        self.m0, self.Ft = engine.dev(m0)[None], engine.dev(F0).T
        self.eps0 = mk(P, p.Ds)
        self.draws = None
        if num_features is not None:
            dyn = pilco.mgpr.device_gp()
            self.feat = (mk(dyn.E, int(num_features), dyn.D), mk(P, dyn.E, 2 * int(num_features)), mk(P, dyn.E, dyn.n))
            self.draws = engine.feature_draws(dyn, P, num_features, *self.feat)
            p.set_inputs(p.x0, None, nu=p.nu_buf if p.nz is not None else None, features=self.draws)
        self.graph, self.stream = None, torch.cuda.Stream()

    def _draw(self, it, base):
        """the draws of one iteration at the counter ``it``, under stream ids base + 0 .. 6"""
        p, s = self.plan, self.seed
        engine.normals(self.eps0, s, base, it)
        p.x0.copy_(self.m0 + self.eps0 @ self.Ft)
        if p.H > 0:
            if self.draws is not None:
                for j, buf in enumerate(self.feat):
                    engine.normals(buf, s, base + 4 + j, it)
                engine.feature_draws(self.pilco.mgpr.device_gp(), p.P, self.draws.F, *self.feat, out=self.draws)
            else:
                engine.normals(p.eps_buf, s, base + 1, it)
            if p.nz is not None:
                engine.normals(p.nu_buf, s, base + 2, it)
            if p.resample:
                engine.normals(p.xi_buf, s, base + 3, it)

    def _evaluate(self, it, base):
        """the draws at ``it``, then the pathwise gradient of every restart at theta, packed -> value [R]"""
        self._draw(it, base)
        th = self._unpack(self.theta, self.plan, self.gp)
        g = self.plan.launch_grad()
        info = self.gp.info if self.gp is not None else torch.zeros_like(g["value"])
        self._pack(self.packed, g["value"].reshape(self.R), info.reshape(self.R), g, th)
        return g["value"].reshape(self.R)

    def iteration(self):
        self._evaluate(self.adam.iter, 0)
        self.adam.step(self.theta, self.packed)

    def restart(self):
        """theta back to the starting points and Adam's state to its start"""
        self.theta.copy_(self.flats0)
        self.adam.reset()

    def capture(self):
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            self.iteration()
            self.restart()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.iteration()
        self.graph = g

    def replay(self):
        with torch.cuda.stream(self.stream):
            self.graph.replay()

    def held_out(self):
        """-> value [R] (device) of the current theta on the held-out sample, enqueued on the group's stream"""
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            value = self._evaluate(self.zero, self.HELD_OUT).clone()
        cur.wait_stream(self.stream)
        return value


def optimize_stochastic(pilco, maxiter, restarts, num_samples, seed, consistent=False, exploration=None,
                        resample=False, num_features=None, measurement_noise=None, lr=1e-3, betas=(0.9, 0.999),
                        eps=1e-8, max_norm=None, flats0=None, m0=None, S0=None):
    """Adam on the sampled return with fresh particles at every step (DESIGN.md section 32).  The restarts start from
    ``flats0`` (default ``initial_flats``), are sharded over ranks with ``shard_restarts`` and dealt to lock-step groups
    (``StochasticEvaluator``), each of which captures one iteration as a CUDA graph and replays it ``maxiter`` times
    with no host synchronisation until the end.  Every restart's final parameters are then scored once on the common
    held-out sample, and the winner is picked by ``gather_table`` + ``select_best`` on [-held-out value | theta].
    ``m0``, ``S0``: the initial state distribution (default pilco.m_init, pilco.S_init).
    Returns (best_flat, best held-out value, per-restart held-out values, trace [maxiter, restarts] of the in-sample
    values, ok [maxiter, restarts]); the trace's columns of restarts on other ranks are NaN (ok False)."""
    from .models.pilco import _sqrt_factor
    maxiter, restarts = int(maxiter), max(int(restarts), 1)
    if maxiter < 1:
        raise ValueError("optimize_stochastic: needs maxiter >= 1 (maxiter=%d)" % maxiter)
    engine.adam_hyperparameters(lr, betas, eps, max_norm)
    dist, rank, world = _dist()
    flats0 = initial_flats(pilco.controller, restarts) if flats0 is None else np.asarray(flats0, dtype=np.float64)
    m0 = np.asarray(pilco.m_init if m0 is None else m0, dtype=np.float64).reshape(-1)
    S0 = np.asarray(pilco.S_init if S0 is None else S0, dtype=np.float64).reshape(m0.size, m0.size)
    F0 = _sqrt_factor(S0)
    mine = shard_restarts(restarts, rank, world)
    P = flats0.shape[1]
    local = np.full((restarts, 1 + P), np.nan)
    trace, ok = np.full((maxiter, restarts), np.nan), np.zeros((maxiter, restarts), dtype=bool)
    if mine:
        bounds = group_bounds(len(mine))
        evs = [StochasticEvaluator(pilco, hi - lo, flats0[mine][lo:hi], num_samples, seed, m0, F0,
                                   consistent=consistent, exploration=exploration, resample=resample,
                                   num_features=num_features, measurement_noise=measurement_noise, lr=lr, betas=betas,
                                   eps=eps, max_norm=max_norm, trace_rows=maxiter) for lo, hi in bounds]
        for ev in evs:
            ev.capture()
        for _ in range(maxiter):
            for ev in evs:
                ev.replay()
        values = [ev.held_out() for ev in evs]
        torch.cuda.synchronize()
        cols = np.asarray(mine)
        for ev, (lo, hi), v in zip(evs, bounds, values):
            local[cols[lo:hi], 0] = -v.cpu().numpy()
            local[cols[lo:hi], 1:] = ev.theta.cpu().numpy()
            trace[:, cols[lo:hi]] = ev.adam.trace.cpu().numpy()
            ok[:, cols[lo:hi]] = ev.adam.ok.cpu().numpy() != 0
        LAST_STATS.update(evals=maxiter, restarts_local=len(mine), horizon=int(pilco.horizon), groups=len(evs),
                          rollout_steps=maxiter * len(mine) * int(pilco.horizon))
    local = gather_table(local, restarts, rank, world, dist)
    best = select_best(local)
    return local[best, 1:], -float(local[best, 0]), [-float(v) for v in local[:, 0]], trace, ok


class CemPolicySearch(_FlatEvaluator):
    """The cross-entropy method over a stationary policy's flat parameter vector (``controller.get_flat()`` layout, n
    long) on the sampled return, every iteration on the device (DESIGN.md section 33).

    ``K`` candidates are rolled out over the same P particles (``engine.ParticleBatchPlan``: x0, eps and, with
    ``measurement_noise``, nu, filled by ``set_inputs``) and scored by their mean return.  A diagonal Gaussian over the
    n parameters, started at the controller's current vector with std ``std0`` (a scalar or [n]), is refitted to the
    ``elites`` best with smoothing ``alpha`` (pilco_cem_update at H = 1, U = n and unbounded candidates).
    ``launch()`` enqueues, with no host synchronisation:
      1. population 0: ``engine.normals`` into xi [K,n] under ``seed`` and stream id ``STREAM`` at iteration 0, then
         pilco_cem_draw (row k = mean + std xi_k, row 0 = mean);
      2. per iteration i: ``_unpack`` of the K rows into the plan's policy buffers (RBF: the batched refactorisation),
         the plan's ``launch()`` (an RBF candidate whose factorisation failed gets a NaN value), the normals of
         population i + 1 at iteration i + 1 (read from a device arange), and pilco_cem_update, which keeps the best
         candidate so far, writes trace row i and draws the next population.
    Row 0 of every population is the mean, so ``best_value`` is never below the start's value on the same particles; a
    candidate with a NaN value ranks last and never becomes the best.  ``run()`` runs ``launch()`` eagerly once (the
    warm-up), captures it as one CUDA graph and replays it once.  Afterwards ``best`` [n] and ``best_value`` [1] hold the
    best candidate and its value, ``mean`` and ``std`` [n] the sampling distribution and ``trace`` [iters,2] each
    iteration's top value and elites' mean value."""

    STREAM = 32              # the candidates' normals (the Adam draws use stream ids 0 .. 6 and 16 .. 22)
    ALPHA = 0.1              # engine.CemPlan's smoothing

    def __init__(self, pilco, K, elites, iters, num_samples, seed, std0=0.5, consistent=False, angles=None,
                 measurement_noise=None, alpha=ALPHA, max_ws_bytes=None):
        super().__init__(pilco, int(K))
        if self.sched:
            raise ValueError("CemPolicySearch: a TimeVaryingLinearController plans with PILCO.plan(optimizer='cem')")
        K, ke, iters, n = self.R, int(elites), int(iters), self.P
        if not 1 <= K <= _lib.CEM_MAX_K or not 1 <= ke <= K or iters < 1:
            raise ValueError("CemPolicySearch: needs 1 <= population <= %d, 1 <= elites <= population and iters >= 1 "
                             "(population=%d, elites=%d, iters=%d)" % (_lib.CEM_MAX_K, K, ke, iters))
        std0 = np.broadcast_to(np.asarray(std0, dtype=np.float64), (n,)).copy()
        if not (np.isfinite(std0).all() and (std0 > 0.0).all()):
            raise ValueError("CemPolicySearch: the initial std must be finite and > 0 (a scalar or %d values)" % n)
        self.K, self.elites, self.iters, self.seed, self.alpha = K, ke, iters, int(seed), float(alpha)
        terms, mult_mu = pilco.reward_spec()
        spec = self.c.policy_spec(self.flat0) if self.linear or self.mlp else pilco.policy_spec(self.flat0)
        self.plan = engine.ParticleBatchPlan(pilco.mgpr.device_gp(), spec, terms, int(num_samples), int(pilco.horizon),
                                             K, mult_mu=mult_mu, consistent=consistent, angles=angles,
                                             measurement_noise=measurement_noise, max_ws_bytes=max_ws_bytes)
        self.gp = self.plan.rbf
        d = engine.device()
        self.mean0, self.std0 = engine.dev(self.flat0[0]), engine.dev(std0)
        self.xi = torch.zeros((K, n), dtype=torch.float64, device=d)
        self.its = torch.arange(iters, dtype=torch.int64, device=d)       # population i's normals: iteration i
        self.loop = engine.CemLoop(K, 1, n, ke, iters, self.alpha, np.inf, self.plan.value, [self.xi] * iters,
                                   self.mean0, self.std0)
        self.cand, self.mean, self.std = self.loop.cand.view(K, n), self.loop.mean.view(n), self.loop.std.view(n)
        self.best, self.best_value, self.trace = self.loop.best.view(n), self.loop.best_value, self.loop.trace
        self.draw, self.updates, self.uws, self.uws_bytes = self.loop.draw, self.loop.updates, self.loop.uws, \
            self.loop.uws_bytes

    def set_inputs(self, x0, eps, nu=None):
        self.plan.set_inputs(x0, eps, nu)

    def evaluate(self):
        """the plan's rollouts of the current population -> value [K]; a candidate whose RBF factorisation failed
        gets NaN"""
        self._unpack(self.cand, self.plan, self.gp)
        value = self.plan.launch()
        if self.gp is not None:
            value.masked_fill_(self.gp.info.reshape(self.K) != 0, float("nan"))
        return value

    def _redraw(self, i):
        """population i's normals: iteration i under ``seed`` and stream id ``STREAM``"""
        engine.normals(self.xi, self.seed, self.STREAM, self.its[i:i + 1])

    def launch(self):
        """the whole search on the current stream, from the start: no host synchronisation"""
        self.loop.launch(self.evaluate, self._redraw)
        return self.best, self.best_value

    def run(self):
        """``launch()`` eagerly (warm-up), then captured as one CUDA graph (``engine.CemLoop.capture``) and replayed
        once -> (best [n], best_value [1]).  The graph is released after its replay."""
        g = self.loop.capture(self.evaluate, self._redraw)
        g.replay()
        torch.cuda.synchronize()
        del g
        return self.best, self.best_value


def _no_box(pilco):
    terms, _ = pilco.reward_spec()
    if any(t["kind"] == _lib.REWARD_BOX for t in terms):
        raise ValueError("the sampled return's pathwise gradient ignores box (risk) terms: their indicator is flat "
                         "almost everywhere, so optimising it would ignore the constraint")


class LockstepLBFGS:
    """R independent SciPy L-BFGS-B runs whose objective evaluations are served in batches."""

    def __init__(self, evaluate, x0, maxiter):
        self.evaluate, self.x = evaluate, np.array(x0, dtype=np.float64)
        self.R = self.x.shape[0]
        self.maxiter = maxiter
        self.cv = threading.Condition()
        self.pending = [False] * self.R
        self.active = [True] * self.R
        self.result = [None] * self.R
        self.generation = 0
        self.final = [None] * self.R
        self.errors = []

    def _worker(self, i):
        def fun(x):
            with self.cv:
                self.x[i] = x
                self.pending[i] = True
                gen = self.generation
                self.cv.notify_all()
                while self.generation == gen:
                    self.cv.wait()
                f, g = self.result[i]
            return f, g
        try:
            res = scipy.optimize.minimize(fun, self.x[i].copy(), jac=True, method="L-BFGS-B",
                                          options=dict(maxiter=self.maxiter))
            self.final[i] = (float(res.fun), np.array(res.x))
        except Exception as exc:          # pragma: no cover
            self.errors.append(exc)
        finally:
            with self.cv:
                self.active[i] = False
                self.cv.notify_all()

    def run(self):
        threads = [threading.Thread(target=self._worker, args=(i,), daemon=True) for i in range(self.R)]
        for t in threads:
            t.start()
        failure = None
        while True:
            with self.cv:
                while any(self.active[i] and not self.pending[i] for i in range(self.R)):
                    self.cv.wait()
                if not any(self.active):
                    break
                xs = self.x.copy()
            if failure is None:
                try:
                    loss, grad = self.evaluate(xs)             # device work happens on this (main) thread
                except BaseException as exc:                   # noqa: BLE001 -- re-raised below, after the workers left
                    failure = exc
            if failure is not None:
                # a failed evaluation (CUDA error, failed check) must not strand the workers in cv.wait():
                # serve (BIG, 0) so that every SciPy instance terminates (flat objective), then re-raise
                loss, grad = np.full(self.R, BIG), np.zeros_like(xs)
            with self.cv:
                for i in range(self.R):
                    if self.pending[i]:
                        self.result[i] = (float(loss[i]), grad[i].copy())
                        self.pending[i] = False
                self.generation += 1
                self.cv.notify_all()
        for t in threads:
            t.join()
        if failure is not None:
            raise failure
        if self.errors:
            raise self.errors[0]
        return self.final


def shard_restarts(restarts, rank, world):
    """restart r -> rank r % world (SURVEY.md section 8e)."""
    return [r for r in range(restarts) if r % world == rank]


def select_best(table):
    """table [restarts, 1+P] = [loss | flat]; lowest loss wins, ties -> lowest restart index."""
    losses = table[:, 0]
    best = int(np.flatnonzero(losses == np.nanmin(losses))[0]) if np.isfinite(losses).any() else 0
    return best


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


def gather_table(local, restarts, rank, world, dist):
    """One all_gather of the per-restart rows ``[loss | flat]`` (NCCL over NVLink on the GPU box, gloo in the
    CPU tests).  Rows of restarts owned by other ranks are NaN on input and filled on output."""
    if world <= 1:
        return local
    P1 = local.shape[1]
    dev = engine.device() if dist.get_backend() == "nccl" else torch.device("cpu")
    per = (restarts + world - 1) // world
    mine = shard_restarts(restarts, rank, world)
    send = torch.full((per, P1), float("nan"), dtype=torch.float64, device=dev)
    if mine:
        send[:len(mine)] = torch.as_tensor(local[mine]).to(dev)
    gathered = [torch.empty_like(send) for _ in range(world)]
    dist.all_gather(gathered, send)                        # the one collective of the hot path
    out = local.copy()
    for g_rank, t in enumerate(gathered):
        rows = shard_restarts(restarts, g_rank, world)
        if rows:
            out[rows] = t[:len(rows)].cpu().numpy()
    return out


def initial_flats(controller, restarts):
    """Restart 0 starts from the current parameters, restarts 1.. from ``controller.randomize()``
    (pilco.py:94-99).  Every rank draws the same sequence from the global numpy RNG."""
    flats = [controller.get_flat()]
    saved = flats[0].copy()
    for _ in range(restarts - 1):
        controller.randomize()
        flats.append(controller.get_flat())
    controller.set_flat(saved)
    return np.stack(flats)


def optimize(pilco, maxiter=50, restarts=1, evaluator=PolicyEvaluator, flats0=None):
    """Returns (best_flat, best_reward, per-restart rewards).  ``evaluator(pilco, R)`` builds the evaluator of one
    lock-step group of R restarts (``PolicyEvaluator``: the moment-matching reward); ``flats0`` [restarts, P] are the
    starting points (default ``initial_flats``)."""
    restarts = max(int(restarts), 1)
    dist, rank, world = _dist()
    flats0 = initial_flats(pilco.controller, restarts) if flats0 is None else np.asarray(flats0, dtype=np.float64)
    mine = shard_restarts(restarts, rank, world)
    P = flats0.shape[1]
    local = np.full((restarts, 1 + P), np.nan)
    if mine:
        x0 = flats0[mine]
        bounds = group_bounds(len(mine))
        evs = [evaluator(pilco, hi - lo) for lo, hi in bounds]
        for ev, (lo, hi) in zip(evs, bounds):
            ev.prepare(x0[lo:hi])
        xs, loss = np.empty_like(x0), np.empty(len(mine))
        errors = []

        def drive(k):
            (lo, hi), ev = bounds[k], evs[k]
            try:
                time.sleep(k * ev.eval_s / len(evs))           # groups out of phase: one sweeps back while the other tiles
                finals = LockstepLBFGS(ev, x0[lo:hi], maxiter).run()
                xs[lo:hi] = np.stack([f[1] for f in finals])
                ev.cache = None
                loss[lo:hi] = ev(xs[lo:hi])[0]                 # rewards at the final points (pilco.py:96,103)
            except BaseException as exc:                       # noqa: BLE001 -- re-raised on the calling thread
                errors.append(exc)
        if len(evs) == 1:
            drive(0)
        else:
            drivers = [threading.Thread(target=drive, args=(k,), daemon=True) for k in range(len(evs))]
            for t in drivers:
                t.start()
            for t in drivers:
                t.join()
        if errors:
            raise errors[0]
        LAST_STATS.update(evals=max(int(ev.ncalls) for ev in evs), restarts_local=len(mine), horizon=int(pilco.horizon),
                          groups=len(evs),
                          rollout_steps=int(sum(ev.ncalls * ev.R for ev in evs)) * int(pilco.horizon))
        for k, r in enumerate(mine):
            local[r, 0] = loss[k]
            local[r, 1:] = xs[k]
    local = gather_table(local, restarts, rank, world, dist)
    best = select_best(local)
    return local[best, 1:], -float(local[best, 0]), [-float(v) for v in local[:, 0]]
