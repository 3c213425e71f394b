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
        self.linear = isinstance(c, controllers.LinearController)
        self.flat0 = np.tile(c.get_flat(), (R, 1))
        self.P = self.flat0.shape[1]
        if self.linear:
            U, Ds = c.W.shape
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

    def _pack(self, out, value, info, g, th):
        """out [R,P+2] = [-value | status | -gradient in the flat layout]; the lengthscale block goes through the
        softplus: d ell / d theta = sigmoid(theta)"""
        R = out.shape[0]
        Ds, U = self.shape
        out[:, 0] = -value
        out[:, 1] = info.to(torch.float64)
        if self.linear:
            out[:, 2:2 + U * Ds] = -g["W"].reshape(R, -1)
            out[:, 2 + U * Ds:] = -g["b"].reshape(R, -1)
        else:
            bf = g["X"].shape[-2]
            out[:, 2:2 + bf * Ds] = -g["X"].reshape(R, -1)
            out[:, 2 + bf * Ds:2 + bf * Ds + bf * U] = -g["Y"].reshape(R, -1)
            out[:, 2 + bf * Ds + bf * U:] = -(g["ell"].reshape(R, U, Ds) * torch.sigmoid(th)).reshape(R, -1)


class PolicyEvaluator(_FlatEvaluator):
    """loss(flat) = -sum_t E[r(x_t)] and its gradient for a batch of flat policy parameter vectors.

    The R restarts are dealt to ``nsplit`` sub-batches, each with its own RolloutPlan (taped forward + reverse sweep)
    on its own stream inside ONE captured CUDA graph: the latency-bound glue kernels of one sub-batch overlap the tile
    kernels of the others."""

    NSPLIT = 4

    def __init__(self, pilco, R, nsplit=None):
        super().__init__(pilco, R)
        c, flat0 = self.c, self.flat0
        terms, mult_mu = pilco.reward_spec()
        nsplit = max(1, min(int(self.NSPLIT if nsplit is None else nsplit), R // 4 if R >= 8 else 1))
        bounds = [round(k * R / nsplit) for k in range(nsplit + 1)]
        self.slices = [(bounds[k], bounds[k + 1]) for k in range(nsplit) if bounds[k + 1] > bounds[k]]
        self.plans, self.gps = [], []
        dyn = pilco.mgpr.device_gp()
        for lo, hi in self.slices:
            spec = c.policy_spec(flat0[lo:hi]) if self.linear else pilco.policy_spec(flat0[lo:hi])
            self.gps.append(None if self.linear else spec["gp"])
            self.plans.append(engine.RolloutPlan(dyn, spec, terms, np.asarray(pilco.m_init, dtype=np.float64).reshape(-1),
                                                 np.asarray(pilco.S_init, dtype=np.float64), int(pilco.horizon), R=hi - lo,
                                                 mult_mu=mult_mu, grad=True))
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
    ``engine.ConsistentGradPlan``).  Box terms carry no pathwise gradient, so a reward with them is rejected."""

    def __init__(self, pilco, R, x0, eps, consistent=False):
        terms, mult_mu = pilco.reward_spec()
        if any(t["kind"] == _lib.REWARD_BOX for t in terms):
            raise ValueError("the sampled return's pathwise gradient ignores box (risk) terms: their indicator is flat "
                             "almost everywhere, so optimising it would ignore the constraint")
        super().__init__(pilco, R)
        c, flat0 = self.c, self.flat0
        spec = c.policy_spec(flat0) if self.linear else pilco.policy_spec(flat0)
        self.gp = None if self.linear else spec["gp"]
        x0 = engine.dev(x0)
        if consistent:
            self.plan = engine.ConsistentGradPlan(pilco.mgpr.device_gp(), spec, terms, int(x0.shape[0]),
                                                  int(pilco.horizon), mult_mu=mult_mu, R=R)
        else:
            self.plan = engine.ParticlePlan(pilco.mgpr.device_gp(), spec, terms, int(x0.shape[0]), int(pilco.horizon),
                                            mult_mu=mult_mu, grad=True, R=R)
        self.plan.set_inputs(x0, eps)
        self._setup_io()

    def _enqueue(self):
        self.d_flat.copy_(self.h_flat, non_blocking=True)
        th = self._unpack(self.d_flat, self.plan, self.gp)
        g = self.plan.launch_grad()
        info = self.gp.info if not self.linear else torch.zeros_like(g["value"])
        self._pack(self.d_out, g["value"].reshape(self.R), info.reshape(self.R), g, th)
        self.h_out.copy_(self.d_out, non_blocking=True)


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
