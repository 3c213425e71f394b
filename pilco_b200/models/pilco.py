"""PILCO orchestrator (drop-in for pilco/models/pilco.py:15-160).

The H-step moment-matching cascade (``predict``/``propagate``, pilco.py:118-153) and the policy
objective with its gradient run on the device through ``pilco_rollout_*``; policy optimisation batches
the random restarts (pilco.py:98-107) in one device rollout and shards them across ranks
(``pilco_b200.policy_opt``)."""
import collections
import time

import numpy as np
import pandas as pd

from .. import controllers, rewards, engine, _lib
from ..params import host, set_trainable
from .mgpr import MGPR
from .smgpr import SMGPR

ParticleTrajectories = collections.namedtuple("ParticleTrajectories", ["states", "actions", "rewards", "risks", "returns"])
ParticlePolicyGradient = collections.namedtuple("ParticlePolicyGradient", ["value", "grad", "returns"])


def _sqrt_factor(S):
    """F with F F' = S: the Cholesky factor, or for a positive semi-definite S (S = 0 included) the eigen-factor
    Q diag(sqrt(max(lambda, 0))).  ValueError when S has an eigenvalue below -1e-12 max|lambda|."""
    import torch
    St = torch.as_tensor(S, dtype=torch.float64)
    L, info = torch.linalg.cholesky_ex(St)
    if int(info) == 0:
        return L.numpy()
    lam, Q = torch.linalg.eigh(St)
    if float(lam.min()) < -1e-12 * float(lam.abs().max()):
        raise ValueError("sample_trajectories: s_x is not positive semi-definite (smallest eigenvalue %.3e)" % float(lam.min()))
    return (Q * lam.clamp(min=0.0).sqrt()[None, :]).numpy()


class PILCO:
    def __init__(self, data, num_induced_points=None, horizon=30, controller=None,
                 reward=None, m_init=None, S_init=None, name=None):
        self.name = name
        if num_induced_points is None:
            self.mgpr = MGPR(data)
        else:
            self.mgpr = SMGPR(data, num_induced_points)
        self.state_dim = data[1].shape[1]
        self.control_dim = data[0].shape[1] - data[1].shape[1]
        self.horizon = horizon
        self.controller = controller if controller is not None else \
            controllers.LinearController(self.state_dim, self.control_dim)
        self.reward = reward if reward is not None else rewards.ExponentialReward(self.state_dim)
        if m_init is None or S_init is None:
            # first state of the data set, pilco.py:36-41
            self.m_init = data[0][0:1, 0:self.state_dim]
            self.S_init = np.diag(np.ones(self.state_dim) * 0.1)
        else:
            self.m_init = m_init
            self.S_init = S_init
        self.optimizer = None

    # ---- parameters ------------------------------------------------------------------------------
    @property
    def trainable_parameters(self):
        return list(self.mgpr.trainable_parameters) + list(self.controller.trainable_parameters)

    # ---- device rollout ---------------------------------------------------------------------------
    def policy_spec(self, flats=None):
        """Description of the policy for ``RolloutPlan``; ``flats`` [R,P] = per-restart flat parameters."""
        c = self.controller
        if isinstance(c, controllers.LinearController):
            return c.policy_spec(flats)
        if isinstance(c, controllers.RbfController):
            bf, Ds, U = c.policy_shapes
            if flats is None:
                gp = c.device_gp()
            else:
                X, Y, th = c.split_flat(flats)
                ell = c.models[0].kernel.lengthscales.transform.forward(th)      # lower + softplus (controllers.py:100)
                R = X.shape[0]
                # kernel variance and noise are the controller's own Parameters (sf2 = 1 and sn2 = 1e-4 unless the
                # user changed them, controllers.py:77-78,91-93) -- the same values compute_reward()/predict() see
                sf2 = np.tile(np.asarray(c.variance, dtype=np.float64).reshape(1, U), (R, 1))
                sn2 = np.tile(np.asarray(c.noise, dtype=np.float64).reshape(1, U), (R, 1))
                gp = engine.gp_factorize(X, Y, ell, sf2, sn2, need_iK=False, mode=1)
            return dict(kind=_lib.POLICY_RBF, Ds=Ds, U=U, squash=True,
                        max_action=controllers._max_action_vec(c.max_action, U), gp=gp)
        raise TypeError("unsupported controller type %r" % type(c))

    def reward_spec(self):
        """(reward terms, mult_mu) handed to the device rollout; SafePILCO adds a multiplicative channel."""
        return self.reward.terms(), 0.0

    def rollout_plan(self, m_x, s_x, n, flats=None):
        R = 1 if flats is None else int(np.asarray(flats).shape[0])
        terms, mult_mu = self.reward_spec()
        return engine.RolloutPlan(self.mgpr.device_gp(), self.policy_spec(flats), terms,
                                  np.asarray(m_x, dtype=np.float64).reshape(-1),
                                  np.asarray(s_x, dtype=np.float64), int(n), R=R, mult_mu=mult_mu)

    def _reward_key(self):
        terms, mult_mu = self.reward_spec()
        parts = [repr(float(mult_mu))]
        for t in terms:
            parts.append(repr((int(t["kind"]), float(t.get("coef", 1.0)), int(t.get("channel", 0)))))
            parts.append(np.ascontiguousarray(np.asarray(t["W"], dtype=np.float64)).tobytes())
            parts.append(b"" if t.get("t") is None else np.ascontiguousarray(np.asarray(t["t"], dtype=np.float64)).tobytes())
        return hash(tuple(parts))

    def _predict_plan(self, n):
        """Captured n-step cascade, cached per (model, policy, reward, n) state: the reference rebuilds nothing
        between calls either (tf.function), but here the cache is explicit -- any change of data, hyper-parameters,
        policy parameters or reward parameters changes the key and rebuilds the plan (a few ms)."""
        dyn = self.mgpr.device_gp()                       # (re)factorises only when data / hypers changed
        key = (id(dyn), self.mgpr._cache_key, self.controller.state_key(), self._reward_key(), int(n))
        cache = self.__dict__.setdefault("_plans", {})
        hit = cache.get(int(n))
        if hit is None or hit[0] != key:
            terms, mult_mu = self.reward_spec()
            plan = engine.PredictPlan(dyn, self.policy_spec(), terms, self.state_dim, int(n), mult_mu=mult_mu)
            if len(cache) >= 8:
                cache.clear()
            cache[int(n)] = hit = (key, plan)
        return hit[1]

    def predict(self, m_x, s_x, n):
        """n-step cascade (pilco.py:118-136) -> (m [1,Ds], S [Ds,Ds], reward [1,1]): one replay of a cached
        CUDA graph (host moments in, host moments out)."""
        from ..params import HostArray
        M, S, rew = self._predict_plan(n)(m_x, s_x)
        return M.view(HostArray), S.view(HostArray), rew.view(HostArray)

    def propagate(self, m_x, s_x):
        """one step (pilco.py:138-153) -> (M_x [1,Ds], S_x [Ds,Ds])"""
        M, S, _ = self.predict(m_x, s_x, 1)
        return M, S

    def sample_trajectories(self, m_x, s_x, n, num_samples=1000, seed=None, consistent=False):
        """Monte Carlo rollouts of the learnt dynamics under the policy, to check what ``predict``'s moment matching
        approximates: ``num_samples`` particles start at x0 ~ N(m_x, s_x) and take n steps of
        x_{t+1} = x_t + mu(x_t, u_t) + sqrt(var(x_t, u_t)) eps_t with the latent GP posterior mean and variance,
        u_t = compute_action(x_t).  Rewards are the reward terms at the particle's state (the expectation of
        ``predict``'s reward is their mean).  Every draw comes from one device ``torch.Generator``; with
        ``seed=None`` its seed is drawn from ``np.random``.  s_x may be singular (a known start state: s_x = 0).

        ``consistent=True``: each particle follows ONE function drawn from the GP posterior, conditioned at every step
        on the particle's own earlier inputs (a state region visited twice has the same dynamics both times), as the
        PILCO papers' sampled trajectories do; the step-wise default draws fresh noise at every step.  The same seed
        gives the same x0 and normals, so step 0 is the same in both.  Its device workspace grows as
        num_samples n^2 (and n times the model's centres); large batches run in chunks.

        -> ParticleTrajectories(states [S,n+1,Ds], actions [S,n,U], rewards [S,n], risks [S,n], returns [S]) of
        host arrays; ``risks`` is the multiplicative channel of SafePILCO (zeros otherwise) and
        returns = rewards.sum(1) (+ mu (1 - prod_t (1 - risks)) for SafePILCO)."""
        from ..params import HostArray
        if consistent:
            import torch
            dyn = self.mgpr.device_gp()
            x0, eps = self._particle_inputs(m_x, s_x, n, num_samples, seed, "sample_trajectories")
            if eps is None:                                     # n = 0
                eps = torch.zeros((int(num_samples), 0, self.state_dim), dtype=engine.F64, device=x0.device)
            terms, mult_mu = self.reward_spec()
            out = engine.particles_rollout(dyn, self.policy_spec(), terms, x0, eps, mult_mu=mult_mu, consistent=True)
            return ParticleTrajectories(*[t.cpu().numpy().view(HostArray) for t in out])
        plan = self._particle_plan(m_x, s_x, n, num_samples, seed, "sample_trajectories")
        plan.launch()
        out = [t.cpu().numpy().view(HostArray) for t in plan.outputs()]
        return ParticleTrajectories(*out)

    def _particle_plan(self, m_x, s_x, n, num_samples, seed, what, grad=False, consistent=False, estimator="pathwise"):
        """ParticlePlan with x0 = m + F eps0 and the step normals drawn from one device generator seeded with ``seed``
        (from ``np.random`` when None): the same seed gives the same particles to every caller.  ``consistent``
        (with ``grad``): the ConsistentGradPlan over the same particles.  ``estimator``: ParticlePlan's."""
        dyn = self.mgpr.device_gp()
        x0, eps = self._particle_inputs(m_x, s_x, n, num_samples, seed, what)
        terms, mult_mu = self.reward_spec()
        if consistent:
            plan = engine.ConsistentGradPlan(dyn, self.policy_spec(), terms, int(num_samples), int(n), mult_mu=mult_mu)
        else:
            plan = engine.ParticlePlan(dyn, self.policy_spec(), terms, int(num_samples), int(n), mult_mu=mult_mu,
                                       grad=grad, estimator=estimator)
        plan.set_inputs(x0, eps)
        return plan

    def _particle_inputs(self, m_x, s_x, n, num_samples, seed, what):
        """(x0 [S,Ds], eps [S,n,Ds]) device tensors of ``_particle_plan``: x0 = m + F eps0, then the step normals, from
        one device generator seeded with ``seed`` (from ``np.random`` when None)."""
        import torch
        n, S = int(n), int(num_samples)
        if n < 0 or S < 1:
            raise ValueError("%s: needs n >= 0 and num_samples >= 1 (n=%d, num_samples=%d)" % (what, n, S))
        Ds = self.state_dim
        m = np.asarray(m_x, dtype=np.float64).reshape(Ds)
        F = _sqrt_factor(np.asarray(s_x, dtype=np.float64).reshape(Ds, Ds))
        d = engine.device()
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        g = torch.Generator(device=d)
        g.manual_seed(int(seed))
        eps0 = torch.randn((S, Ds), dtype=engine.F64, device=d, generator=g)
        x0 = engine.dev(m)[None] + eps0 @ engine.dev(F).T
        eps = torch.randn((S, n, Ds), dtype=engine.F64, device=d, generator=g) if n > 0 else None
        return x0, eps

    def _flat_grad(self, g):
        """policy gradient blocks (device tensors) -> d / d controller.get_flat(): the lengthscale block times the
        derivative of the softplus transform, sigmoid(theta), as policy_opt applies it"""
        c = self.controller
        if isinstance(c, controllers.LinearController):
            return np.concatenate([g["W"].cpu().numpy().ravel(), g["b"].cpu().numpy().ravel()])
        bf, Ds, U = c.policy_shapes
        th = c.get_flat()[bf * Ds + bf * U:]
        return np.concatenate([g["X"].cpu().numpy().ravel(), g["Y"].cpu().numpy().ravel(),
                               g["ell"].cpu().numpy().ravel() / (1.0 + np.exp(-th))])

    def sample_policy_gradient(self, m_x, s_x, n, num_samples=1000, seed=None, consistent=False, estimator="pathwise"):
        """Pathwise (reparameterisation) gradient of the Monte Carlo return of ``sample_trajectories``: the particles
        are drawn exactly as there (the same seed gives the same particles), value = mean of their returns, and grad =
        d value / d controller.get_flat() with x0 and the step normals held fixed -- the ascent direction of the
        sampled return, to compare with ``policy_gradient``.  Box (risk) terms enter value but not grad: their
        indicator is flat almost everywhere, so for them the estimate of d E[return] is biased.  ``consistent=True``:
        the particles of ``sample_trajectories(..., consistent=True)``, each following one function drawn from the
        dynamics posterior (DESIGN.md section 15); its workspace grows as num_samples n E N (N training points)
        and is not chunked.

        ``estimator="score"``: the score-function (likelihood-ratio) estimate over the same particles instead (DESIGN.md
        section 16), with a leave-one-out baseline.  It differentiates no trajectory, so box terms enter grad and the
        estimate is unbiased for every reward; value and returns are the pathwise call's.  Its variance scales as
        1 / sigma^2 where the model is confident (a small predicted variance), so it can need many more samples than
        the pathwise estimate on smooth rewards.  ``consistent=True`` with ``estimator="score"`` is a ValueError.

        -> ParticlePolicyGradient(value (float), grad [len(get_flat())], returns [num_samples]) host arrays."""
        from ..params import HostArray
        if estimator not in engine.ParticlePlan.ESTIMATORS:
            raise ValueError("sample_policy_gradient: estimator must be one of %s, not %r"
                             % (engine.ParticlePlan.ESTIMATORS, estimator))
        if consistent and estimator == "score":
            raise ValueError("sample_policy_gradient: the score-function estimator is not available for the consistent "
                             "(function-sample) particles; use estimator='pathwise'")
        plan = self._particle_plan(m_x, s_x, n, num_samples, seed, "sample_policy_gradient", grad=True,
                                   consistent=consistent, estimator=estimator)
        g = plan.launch_grad()
        return ParticlePolicyGradient(float(g["value"].item()), self._flat_grad(g).view(HostArray),
                                      plan.ret.cpu().numpy().view(HostArray))

    def policy_gradient(self, m_x=None, s_x=None, n=None):
        """The moment-matching reward of ``predict`` (n steps from N(m_x, s_x); defaults m_init, S_init, horizon) and
        its gradient d reward / d controller.get_flat() for the current policy: the direction ``optimize_policy``
        ascends, in the layout of ``sample_policy_gradient``.  -> (reward (float), grad host array)."""
        from ..params import HostArray
        m_x = self.m_init if m_x is None else m_x
        s_x = self.S_init if s_x is None else s_x
        n = self.horizon if n is None else n
        terms, mult_mu = self.reward_spec()
        plan = engine.RolloutPlan(self.mgpr.device_gp(), self.policy_spec(), terms,
                                  np.asarray(m_x, dtype=np.float64).reshape(-1), np.asarray(s_x, dtype=np.float64),
                                  int(n), R=1, mult_mu=mult_mu, grad=True)
        plan.forward()
        g = plan.backward()
        return float(plan.reward[0].item()), self._flat_grad({k: v[0] for k, v in g.items()}).view(HostArray)

    def optimize_policy_sampled(self, maxiter=50, restarts=1, num_samples=1000, seed=None, consistent=False):
        """Optimise the policy on the sampled return instead of the moment-matching reward (Deep PILCO, PIPPS): the
        objective is the mean return of ``num_samples`` particle rollouts of the learnt dynamics from N(m_init, S_init)
        over ``horizon`` steps, with x0 and the step normals drawn once, exactly as ``sample_trajectories`` and
        ``sample_policy_gradient`` draw them for the same ``seed`` (from ``np.random`` when None, drawn after the
        restarts' starting points).  With the random numbers held fixed the objective is a deterministic, smooth
        function of the policy parameters, which is why L-BFGS-B applies; its gradient is the pathwise one of
        ``sample_policy_gradient``.  Restarts are chosen, batched, sharded over ranks and selected as in
        ``optimize_policy``, evaluated on the same particles.  The controller is set to the winner.

        Returns the winner's sampled value: an in-sample estimate, biased upwards by the optimisation; for an
        out-of-sample estimate run ``sample_trajectories`` with another seed.  A reward with box (risk) terms is
        rejected, because they carry no pathwise gradient and the optimiser would ignore the constraint.

        ``consistent=True``: the particles follow one function drawn from the dynamics posterior each, as
        ``sample_trajectories(..., consistent=True)`` (Deep PILCO's objective), so model errors do not average out
        along a trajectory.  A lock-step group's workspace is O(restarts num_samples horizon^2 E n); a group that
        needs more than half the free device memory is a ValueError naming the num_samples that would fit."""
        from functools import partial
        from .. import policy_opt
        if int(num_samples) < 1:
            raise ValueError("optimize_policy_sampled: needs num_samples >= 1 (num_samples=%d)" % int(num_samples))
        terms, _ = self.reward_spec()
        if any(t["kind"] == _lib.REWARD_BOX for t in terms):
            raise ValueError("optimize_policy_sampled: the reward has box (risk) terms, which carry no pathwise "
                             "gradient; use optimize_policy")
        restarts = max(int(restarts), 1)
        mgpr_trainable = self.mgpr.trainable_parameters
        for p in mgpr_trainable:
            set_trainable(p, False)
        try:
            flats0 = policy_opt.initial_flats(self.controller, restarts)
            x0, eps = self._particle_inputs(self.m_init, self.S_init, self.horizon, num_samples, seed,
                                            "optimize_policy_sampled")
            best_flat, best_value, _ = policy_opt.optimize(
                self, maxiter=maxiter, restarts=restarts, flats0=flats0,
                evaluator=partial(policy_opt.ParticleEvaluator, x0=x0, eps=eps, consistent=consistent))
            self.controller.set_flat(best_flat)
        finally:
            for p in mgpr_trainable:
                set_trainable(p, True)
        return best_value

    def training_loss(self):
        return -self.predict(self.m_init, self.S_init, self.horizon)[2]

    def compute_reward(self):
        return -self.training_loss()

    @property
    def maximum_log_likelihood_objective(self):
        return -self.training_loss()

    def compute_action(self, x_m):
        """pilco.py:115-116: the policy mean at a deterministic state (s = 0).  Served by a cached
        ``engine.ActionPlan`` (one captured CUDA graph per policy state) -- the per-control-step call of
        examples/utils.py:32-36."""
        from ..params import HostArray
        key = self.controller.state_key()
        if key != getattr(self, "_act_key", None):
            self._act_plan = engine.ActionPlan(self.policy_spec())
            self._act_key = key
        return self._act_plan(x_m).view(HostArray)

    # ---- model training (pilco.py:52-73) ------------------------------------------------------------
    def optimize_models(self, maxiter=200, restarts=1):
        self.mgpr.optimize(restarts=restarts)
        lengthscales, variances, noises = {}, {}, {}
        for i, model in enumerate(self.mgpr.models):
            lengthscales['GP' + str(i)] = model.kernel.lengthscales.numpy()
            variances['GP' + str(i)] = np.array([model.kernel.variance.numpy()])
            noises['GP' + str(i)] = np.array([model.likelihood.variance.numpy()])
        print('-----Learned models------')
        pd.set_option('display.precision', 3)
        print('---Lengthscales---')
        print(pd.DataFrame(data=lengthscales))
        print('---Variances---')
        print(pd.DataFrame(data=variances))
        print('---Noises---')
        print(pd.DataFrame(data=noises))

    # ---- policy optimisation (pilco.py:75-113) --------------------------------------------------------
    def optimize_policy(self, maxiter=50, restarts=1):
        from .. import policy_opt
        start = time.time()
        mgpr_trainable = self.mgpr.trainable_parameters
        for p in mgpr_trainable:
            set_trainable(p, False)
        try:
            best_flat, best_reward, all_rewards = policy_opt.optimize(self, maxiter=maxiter, restarts=restarts)
            self.controller.set_flat(best_flat)
        finally:
            for p in mgpr_trainable:
                set_trainable(p, True)
        end = time.time()
        for rwd in all_rewards:
            print("Controller's optimization: done in %.1f seconds with reward=%.3f." % (end - start, rwd))
        return best_reward
