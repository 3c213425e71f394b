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
AdamTrace = collections.namedtuple("AdamTrace", ["value", "ok"])


def _resample_refusals(what, resample, consistent, estimator="pathwise", exploration=0.0):
    """the Gaussian refit's refusals at the class level, as engine.ParticlePlan's (ValueError)"""
    if not resample:
        return
    for on, why in ((consistent, "consistent=True"), (estimator == "score", "estimator='score'"),
                    (float(exploration) != 0.0, "exploration")):
        if on:
            raise ValueError("%s: resample=True does not combine with %s" % (what, why))


def _feature_refusals(what, num_features, consistent, model, estimator="pathwise"):
    """the random-feature sampler's refusals at the class level (ValueError), before any device work: it draws whole
    functions (consistent=True), from the exact GP (not SMGPR's FITC), for the pathwise estimator, with 1 .. 8192
    frequency pairs"""
    if num_features is None:
        return None
    for on, why in ((not consistent, "consistent=False (the draws are whole functions: pass consistent=True)"),
                    (isinstance(model, SMGPR), "an SMGPR (FITC) dynamics model"),
                    (estimator == "score", "estimator='score' (a function sample has no per-step path density)")):
        if on:
            raise ValueError("%s: num_features does not combine with %s" % (what, why))
    F = int(num_features)
    if F < 1 or F > _lib.MAX_FEATURES:
        raise ValueError("%s: num_features must be in 1 .. %d, got %d" % (what, _lib.MAX_FEATURES, F))
    return F


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


def _controller_input_dim(c):
    if isinstance(c, controllers.RbfController):
        return int(c.policy_shapes[1])
    if isinstance(c, (controllers.LinearController, controllers.TimeVaryingLinearController)):
        return int(np.asarray(c.W).shape[-1])
    if isinstance(c, controllers.MlpController):
        return c.state_dim
    return None


class PILCO:
    def __init__(self, data, num_induced_points=None, horizon=30, controller=None,
                 reward=None, m_init=None, S_init=None, name=None, *, angle_dims=None, exploration=0.0,
                 measurement_noise=None):
        """``angle_dims``: angular state dimensions (PILCO's trigonometric augmentation, DESIGN.md section 19).  The
        policy and the dynamics GPs then see phi(x) = [the other state dimensions, sin and cos of each angle] (Dh =
        state_dim + len(angle_dims)), while the state, m_init / S_init, the state reward terms and the GP outputs stay
        raw.  ``data`` stays the raw (X = [x, u], Y = delta x); the angles' deltas in Y must be continuous (unwrapped).
        The models are trained on [phi(x), u], so ``mgpr.models[e].predict_*`` take such inputs; new raw data goes
        through ``PILCO.set_data``.  The controller must take Dh inputs and every joint state-action reward term must
        have state_dim = Dh (ValueError otherwise).

        ``exploration``: the weight b of the original PILCO's exploration objective sum_t (E[r_t] + b sigma_t), sigma_t
        the standard deviation of step t's reward under the predicted state distribution (DESIGN.md section 21).  b > 0
        is optimistic under model uncertainty and draws the policy to states the model does not know; b < 0 is
        risk-averse.  ``optimize_policy``, ``policy_gradient``, ``training_loss`` and ``compute_reward`` use it;
        ``predict`` keeps returning the expected reward.  A plain attribute: reassign ``pilco.exploration`` between
        calls.  A reward with an additive box term has no variance closed form: b != 0 with one is a ValueError.

        ``measurement_noise``: the policy acts on a noisy measurement z = x + nu of the state, nu ~ N(0, diag(v)), as
        on the real system (the original PILCO's propagate.m; DESIGN.md section 22).  The moment-matching methods
        (``predict``, ``propagate``, ``training_loss``, ``compute_reward``, ``policy_gradient``,
        ``predict_reward_moments``, ``optimize_policy``) then moment-match the policy at N(m, S + diag(v)) while the
        dynamics see the true state.  ``None``: the policy sees the state; an array v [state_dim] >= 0 (raw state
        dimensions, angles included); or ``"model"``: v = the dynamics GPs' noise variances / 2 (a difference target
        carries the noise of two measurements), read again at every call, so it follows ``optimize_models``.
        ``compute_action`` is unchanged: on the system it is given the measurement.  The particle methods do not
        support it (ValueError)."""
        self.name = name
        self.exploration = float(exploration)
        self.state_dim = data[1].shape[1]
        self.control_dim = data[0].shape[1] - data[1].shape[1]
        self.angle_dims = None
        if angle_dims is not None and len(angle_dims) > 0:
            engine.angles_struct(angle_dims, self.state_dim)            # ValueError: out of range or repeated
            self.angle_dims = [int(a) for a in angle_dims]
            if self.policy_input_dim + self.control_dim > _lib.ABI_MAX_D:
                raise ValueError("angle_dims: state_dim + %d angles + control_dim = %d exceeds %d"
                                 % (len(self.angle_dims), self.policy_input_dim + self.control_dim, _lib.ABI_MAX_D))
        gp_data = self._model_data(data)
        if num_induced_points is None:
            self.mgpr = MGPR(gp_data)
        else:
            self.mgpr = SMGPR(gp_data, num_induced_points)
        if self.angle_dims is not None:
            self.mgpr._input_width = self.policy_input_dim + self.control_dim
        self.horizon = horizon
        self.controller = controller if controller is not None else \
            controllers.LinearController(self.policy_input_dim, self.control_dim)
        self.reward = reward if reward is not None else rewards.ExponentialReward(self.state_dim)
        if self.angle_dims is not None:
            Dh = self.policy_input_dim
            cin = _controller_input_dim(self.controller)
            if cin is not None and cin != Dh:
                raise ValueError("with angle_dims=%s the controller must take Dh = %d inputs (phi(x)), it takes %d"
                                 % (self.angle_dims, Dh, cin))
            for k, t in enumerate(self.reward.terms()):
                if t["kind"] in _lib.JOINT_REWARDS and int(t.get("state_dim", -1)) != Dh:
                    raise ValueError("with angle_dims=%s reward term %d on the joint [phi(x), u] needs state_dim = Dh = "
                                     "%d, got %s" % (self.angle_dims, k, Dh, t.get("state_dim")))
        if m_init is None or S_init is None:
            # first state of the data set, pilco.py:36-41
            self.m_init = data[0][0:1, 0:self.state_dim]
            self.S_init = np.diag(np.ones(self.state_dim) * 0.1)
        else:
            self.m_init = m_init
            self.S_init = S_init
        self.optimizer = None
        self.measurement_noise = self._check_noise(measurement_noise)

    # ---- measurement noise ---------------------------------------------------------------------------
    def _check_noise(self, v):
        if v is None or (isinstance(v, str) and v == "model"):
            return v
        if isinstance(v, str):
            raise ValueError("measurement_noise: expected None, 'model' or %d variances, got %r" % (self.state_dim, v))
        a = np.asarray(v, dtype=np.float64).reshape(-1)
        if a.shape[0] != self.state_dim or not np.all(np.isfinite(a)) or np.any(a < 0.0):
            raise ValueError("measurement_noise: expected %d finite variances >= 0, got %r" % (self.state_dim, v))
        return a.copy()

    def _noise_var(self):
        """the measurement-noise variances [state_dim] the device rollout gets, or None"""
        v = self.measurement_noise
        if v is None:
            return None
        if isinstance(v, str):                            # "model": propagate.m's sn2(difi) / 2
            return np.asarray(self.mgpr.noise, dtype=np.float64).reshape(-1) / 2.0
        return np.asarray(v, dtype=np.float64)

    def _no_noise(self, what):
        if self.measurement_noise is not None:
            raise ValueError("%s: the particle rollouts do not support measurement_noise yet; use the moment-matching "
                             "methods (predict, policy_gradient, optimize_policy)" % what)

    # ---- angular state dimensions ------------------------------------------------------------------
    @property
    def policy_input_dim(self):
        """Dh: the dimension of what the policy and the dynamics GPs see of the state (state_dim without angles)"""
        return self.state_dim + (len(self.angle_dims) if self.angle_dims else 0)

    def _model_data(self, data):
        """raw (X = [x, u], Y) -> the dynamics GPs' data ([phi(x), u], Y)"""
        if not self.angle_dims:
            return data
        X = np.asarray(data[0], dtype=np.float64)
        Ds = self.state_dim
        return (np.hstack([engine.trig_feature_map(X[:, :Ds], self.angle_dims), X[:, Ds:]]), data[1])

    def set_data(self, data):
        """New raw data (X = [x, u], Y = delta x) for the dynamics GPs; with angle_dims, phi is applied to x."""
        self.mgpr.set_data(self._model_data(data))

    # ---- time-varying linear policy (receding-horizon planning) ------------------------------------
    def _scheduled(self, n=None):
        """True for a TimeVaryingLinearController (the rollouts take schedule=True); an n-step rollout beyond its
        horizon is a ValueError"""
        c = self.controller
        if not isinstance(c, controllers.TimeVaryingLinearController):
            return False
        if n is not None and int(n) > c.horizon:
            raise ValueError("a rollout of n=%d steps runs beyond the TimeVaryingLinearController's horizon of %d steps"
                             % (int(n), c.horizon))
        return True

    def _no_schedule(self, what):
        if isinstance(self.controller, controllers.TimeVaryingLinearController):
            raise ValueError("%s: the particle rollouts do not support the TimeVaryingLinearController; use the "
                             "moment-matching methods (predict, policy_gradient, optimize_policy, plan)" % what)

    def _no_mlp(self, what):
        """the moment-matching methods refuse an MlpController (no closed-form moments), before any device work"""
        if isinstance(self.controller, controllers.MlpController):
            raise TypeError("%s: an MlpController has no moment-matching closed form; train it on the sampled return "
                            "with optimize_policy_sampled (and inspect it with sample_trajectories)" % what)

    def _no_angles(self, what):
        if self.angle_dims:
            raise ValueError("%s: the particle rollouts do not support angle_dims yet; use the moment-matching methods "
                             "(predict, policy_gradient, optimize_policy)" % what)

    # ---- parameters ------------------------------------------------------------------------------
    @property
    def trainable_parameters(self):
        return list(self.mgpr.trainable_parameters) + list(self.controller.trainable_parameters)

    # ---- device rollout ---------------------------------------------------------------------------
    def policy_spec(self, flats=None):
        """Description of the policy for ``RolloutPlan``; ``flats`` [R,P] = per-restart flat parameters."""
        c = self.controller
        if isinstance(c, (controllers.LinearController, controllers.TimeVaryingLinearController,
                          controllers.MlpController)):
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
        self._no_mlp("rollout_plan")
        R = 1 if flats is None else int(np.asarray(flats).shape[0])
        terms, mult_mu = self.reward_spec()
        return engine.RolloutPlan(self.mgpr.device_gp(), self.policy_spec(flats), terms,
                                  np.asarray(m_x, dtype=np.float64).reshape(-1),
                                  np.asarray(s_x, dtype=np.float64), int(n), R=R, mult_mu=mult_mu, angles=self.angle_dims,
                                  measurement_noise=self._noise_var(), schedule=self._scheduled(n))

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
        sched = self._scheduled(n)
        dyn = self.mgpr.device_gp()                       # (re)factorises only when data / hypers changed
        v = self._noise_var()
        key = (id(dyn), self.mgpr._cache_key, self.controller.state_key(), self._reward_key(), int(n),
               None if v is None else v.tobytes())
        cache = self.__dict__.setdefault("_plans", {})
        hit = cache.get(int(n))
        if hit is None or hit[0] != key:
            terms, mult_mu = self.reward_spec()
            plan = engine.PredictPlan(dyn, self.policy_spec(), terms, self.state_dim, int(n), mult_mu=mult_mu,
                                      angles=self.angle_dims, measurement_noise=v, schedule=sched)
            if len(cache) >= 8:
                cache.clear()
            cache[int(n)] = hit = (key, plan)
        return hit[1]

    def predict(self, m_x, s_x, n):
        """n-step cascade (pilco.py:118-136) -> (m [1,Ds], S [Ds,Ds], reward [1,1]): one replay of a cached
        CUDA graph (host moments in, host moments out)."""
        self._no_mlp("predict")
        from ..params import HostArray
        M, S, rew = self._predict_plan(n)(m_x, s_x)
        return M.view(HostArray), S.view(HostArray), rew.view(HostArray)

    def propagate(self, m_x, s_x):
        """one step (pilco.py:138-153) -> (M_x [1,Ds], S_x [Ds,Ds])"""
        self._no_mlp("propagate")
        M, S, _ = self.predict(m_x, s_x, 1)
        return M, S

    def sample_trajectories(self, m_x, s_x, n, num_samples=1000, seed=None, consistent=False, resample=False,
                            num_features=None):
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

        ``resample=True``: Deep PILCO's Gaussian refit (DESIGN.md section 26): at every step the particles are replaced
        by draws from the Gaussian fitted to them (their sample mean and covariance), with standard normals drawn from
        the same generator after the step normals, so a seed gives the same x0 and step normals with and without it.
        It needs num_samples >= 2; with ``consistent=True`` it is a ValueError.

        ``num_features=F`` with ``consistent=True``: each particle's functions are drawn once as a prior of F random
        Fourier features plus an exact data update (DESIGN.md section 30), in time linear in n and with a workspace
        that does not grow with the model's centres.  The same seed gives the same x0; the draws' normals (the
        frequencies, the feature weights, the update's noise) follow from the same generator.  ``None``: the exact
        sampler.  With ``consistent=False`` or an SMGPR model it is a ValueError.

        -> ParticleTrajectories(states [S,n+1,Ds], actions [S,n,U], rewards [S,n], risks [S,n], returns [S]) of
        host arrays; ``risks`` is the multiplicative channel of SafePILCO (zeros otherwise) and
        returns = rewards.sum(1) (+ mu (1 - prod_t (1 - risks)) for SafePILCO)."""
        from ..params import HostArray
        self._no_schedule("sample_trajectories")
        self._no_angles("sample_trajectories")
        self._no_noise("sample_trajectories")
        _resample_refusals("sample_trajectories", resample, consistent)
        F = _feature_refusals("sample_trajectories", num_features, consistent, self.mgpr)
        if F is not None:
            out = self._feature_rollout(m_x, s_x, n, num_samples, seed, F, "sample_trajectories")
            return ParticleTrajectories(*[t.cpu().numpy().view(HostArray) for t in out])
        if consistent:
            import torch
            dyn = self.mgpr.device_gp()
            x0, eps = self._particle_inputs(m_x, s_x, n, num_samples, seed, "sample_trajectories")
            if eps is None:                                     # n = 0
                eps = torch.zeros((int(num_samples), 0, self.state_dim), dtype=engine.F64, device=x0.device)
            terms, mult_mu = self.reward_spec()
            out = engine.particles_rollout(dyn, self.policy_spec(), terms, x0, eps, mult_mu=mult_mu, consistent=True)
            return ParticleTrajectories(*[t.cpu().numpy().view(HostArray) for t in out])
        plan = self._particle_plan(m_x, s_x, n, num_samples, seed, "sample_trajectories", resample=resample)
        plan.launch()
        out = [t.cpu().numpy().view(HostArray) for t in plan.outputs()]
        return ParticleTrajectories(*out)

    def _particle_plan(self, m_x, s_x, n, num_samples, seed, what, grad=False, consistent=False, estimator="pathwise",
                       exploration=None, resample=False, num_features=None):
        """ParticlePlan with x0 = m + F eps0 and the step normals drawn from one device generator seeded with ``seed``
        (from ``np.random`` when None): the same seed gives the same particles to every caller.  ``consistent``
        (with ``grad``): the ConsistentGradPlan over the same particles.  ``estimator``, ``exploration``,
        ``resample``: ParticlePlan's (the redraw's normals come after the step normals).  ``num_features`` (with
        ``consistent`` and ``grad``): the ConsistentGradPlan of the random-feature sampler over ``_feature_inputs``."""
        dyn = self.mgpr.device_gp()
        if num_features is not None:
            x0, draws = self._feature_inputs(m_x, s_x, n, num_samples, seed, num_features, what)
            terms, mult_mu = self.reward_spec()
            plan = engine.ConsistentGradPlan(dyn, self.policy_spec(), terms, int(num_samples), int(n), mult_mu=mult_mu,
                                             exploration=exploration, num_features=num_features)
            plan.set_inputs(x0, None, features=draws)
            return plan
        inputs = self._particle_inputs(m_x, s_x, n, num_samples, seed, what, resample)
        x0, eps, xi = inputs if resample else inputs + (None,)
        terms, mult_mu = self.reward_spec()
        if consistent:
            plan = engine.ConsistentGradPlan(dyn, self.policy_spec(), terms, int(num_samples), int(n), mult_mu=mult_mu,
                                             exploration=exploration)
        else:
            plan = engine.ParticlePlan(dyn, self.policy_spec(), terms, int(num_samples), int(n), mult_mu=mult_mu,
                                       grad=grad, estimator=estimator, exploration=exploration, resample=resample)
        plan.set_inputs(x0, eps, xi=xi)
        return plan

    def _start_states(self, m_x, s_x, S, seed):
        """(x0 = m + F eps0 [S,Ds], the device generator seeded with ``seed`` (from ``np.random`` when None) after
        eps0): the first draws of every particle method"""
        import torch
        Ds = self.state_dim
        m = np.asarray(m_x, dtype=np.float64).reshape(Ds)
        F = _sqrt_factor(np.asarray(s_x, dtype=np.float64).reshape(Ds, Ds))
        d = engine.device()
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        g = torch.Generator(device=d)
        g.manual_seed(int(seed))
        eps0 = torch.randn((S, Ds), dtype=engine.F64, device=d, generator=g)
        return engine.dev(m)[None] + eps0 @ engine.dev(F).T, g

    def _particle_inputs(self, m_x, s_x, n, num_samples, seed, what, resample=False):
        """(x0 [S,Ds], eps [S,n,Ds]) device tensors of ``_particle_plan``: x0 = m + F eps0, then the step normals, from
        one device generator seeded with ``seed`` (from ``np.random`` when None); eps is None at n = 0.  ``resample``:
        (x0, eps, xi), the redraw's normals xi [S,n,Ds] drawn after the step normals from the same generator."""
        import torch
        n, S = int(n), int(num_samples)
        if n < 0 or S < 1:
            raise ValueError("%s: needs n >= 0 and num_samples >= 1 (n=%d, num_samples=%d)" % (what, n, S))
        Ds = self.state_dim
        x0, g = self._start_states(m_x, s_x, S, seed)
        d = x0.device
        eps = torch.randn((S, n, Ds), dtype=engine.F64, device=d, generator=g) if n > 0 else None
        if not resample:
            return x0, eps
        xi = torch.randn((S, n, Ds), dtype=engine.F64, device=d, generator=g) if n > 0 else \
            torch.zeros((S, 0, Ds), dtype=engine.F64, device=d)
        return x0, eps, xi

    def _feature_inputs(self, m_x, s_x, n, num_samples, seed, F, what):
        """(x0 [S,Ds], draws) of the random-feature sampler: x0 exactly as ``_particle_inputs`` draws it for the same
        seed, then from the same generator zeta [E,F,D], w [S,E,2F] and eps_y [S,E,N] (N training points), which
        ``engine.feature_draws`` turns into the draws; no step normals are drawn"""
        import torch
        n, S = int(n), int(num_samples)
        if n < 0 or S < 1:
            raise ValueError("%s: needs n >= 0 and num_samples >= 1 (n=%d, num_samples=%d)" % (what, n, S))
        dyn = self.mgpr.device_gp()
        x0, g = self._start_states(m_x, s_x, S, seed)
        d = x0.device
        zeta = torch.randn((dyn.E, F, dyn.D), dtype=engine.F64, device=d, generator=g)
        w = torch.randn((S, dyn.E, 2 * F), dtype=engine.F64, device=d, generator=g)
        eps_y = torch.randn((S, dyn.E, dyn.n), dtype=engine.F64, device=d, generator=g)
        return x0, engine.feature_draws(dyn, S, F, zeta, w, eps_y)

    def _feature_rollout(self, m_x, s_x, n, num_samples, seed, F, what):
        """the random-feature sampler's forward outputs over ``_feature_inputs``'s particles (chunked when large)"""
        x0, draws = self._feature_inputs(m_x, s_x, n, num_samples, seed, F, what)
        terms, mult_mu = self.reward_spec()
        return engine.particles_rollout(self.mgpr.device_gp(), self.policy_spec(), terms, x0, None, mult_mu=mult_mu,
                                        consistent=True, features=draws, horizon=int(n))

    def _flat_grad(self, g):
        """policy gradient blocks (device tensors) -> d / d controller.get_flat(): the lengthscale block times the
        derivative of the softplus transform, sigmoid(theta), as policy_opt applies it"""
        c = self.controller
        if isinstance(c, controllers.MlpController):
            return g["theta"].cpu().numpy().ravel()
        if isinstance(c, controllers.TimeVaryingLinearController):
            return c.flat_grad(g["W"].cpu().numpy(), g["b"].cpu().numpy())
        if isinstance(c, controllers.LinearController):
            return np.concatenate([g["W"].cpu().numpy().ravel(), g["b"].cpu().numpy().ravel()])
        bf, Ds, U = c.policy_shapes
        th = c.get_flat()[bf * Ds + bf * U:]
        return np.concatenate([g["X"].cpu().numpy().ravel(), g["Y"].cpu().numpy().ravel(),
                               g["ell"].cpu().numpy().ravel() / (1.0 + np.exp(-th))])

    def sample_reward_moments(self, m_x, s_x, n, num_samples=1000, seed=None, consistent=False, resample=False,
                              num_features=None):
        """Sample mean and variance of each step's reward over the particles of ``sample_trajectories`` (the same seed
        gives the same particles): the sampled counterpart of ``predict_reward_moments``.  mean_t is the mean of the
        step rewards (``sample_trajectories(...).rewards.mean(0)`` up to rounding) and var_t = sum_k c_k^2 s_kt^2 over
        the additive terms, s_kt^2 the unbiased sample variance of term k at step t (covariances between terms ignored,
        as ``predict_reward_moments``; the multiplicative terms of SafePILCO do not enter; DESIGN.md section 24).
        ``consistent``: the particles of ``sample_trajectories(..., consistent=True)``; a chunked rollout gives the
        statistics of all num_samples particles.  ``resample``: the particles of ``sample_trajectories(...,
        resample=True)``.  ``num_features``: the particles of ``sample_trajectories(..., consistent=True,
        num_features=F)``.  Needs num_samples >= 2; a reward with an additive box term is a ValueError.  -> (mean [n],
        var [n]) host arrays."""
        from ..params import HostArray
        self._no_schedule("sample_reward_moments")
        self._no_angles("sample_reward_moments")
        self._no_noise("sample_reward_moments")
        _resample_refusals("sample_reward_moments", resample, consistent)
        F = _feature_refusals("sample_reward_moments", num_features, consistent, self.mgpr)
        if int(num_samples) < 2:
            raise ValueError("sample_reward_moments: the sample variance needs num_samples >= 2 (num_samples=%d)"
                             % int(num_samples))
        terms, mult_mu = self.reward_spec()
        engine._no_additive_box(terms)
        if F is not None:
            out = self._feature_rollout(m_x, s_x, n, num_samples, seed, F, "sample_reward_moments")
        elif consistent:
            import torch
            x0, eps = self._particle_inputs(m_x, s_x, n, num_samples, seed, "sample_reward_moments")
            if eps is None:                                     # n = 0
                eps = torch.zeros((int(num_samples), 0, self.state_dim), dtype=engine.F64, device=x0.device)
            out = engine.particles_rollout(self.mgpr.device_gp(), self.policy_spec(), terms, x0, eps, mult_mu=mult_mu,
                                           consistent=True)
        else:
            plan = self._particle_plan(m_x, s_x, n, num_samples, seed, "sample_reward_moments", resample=resample)
            plan.launch()
            out = plan.outputs()
        mean, var = engine.particle_reward_moments(terms, out[0], out[1])
        return mean.cpu().numpy().view(HostArray), var.cpu().numpy().view(HostArray)

    def sample_policy_gradient(self, m_x, s_x, n, num_samples=1000, seed=None, consistent=False, estimator="pathwise",
                               exploration=0.0, resample=False, num_features=None):
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

        ``exploration``: a weight b != 0 makes value PILCO's exploration objective over the particles, mean return +
        b sum_t sigma_t, sigma_t the sample spread of step t's reward (``sample_reward_moments``), and grad its pathwise
        gradient (DESIGN.md section 24).  It does not read ``self.exploration``: pass ``exploration=self.exploration``
        for the sampled counterpart of ``optimize_policy``'s objective.  b != 0 needs num_samples >= 2, the pathwise
        estimator and no additive box term (ValueError otherwise); b = 0 is the call without it.

        ``resample=True``: the particles of ``sample_trajectories(..., resample=True)`` and the pathwise gradient through
        the Gaussian refit, its normals held fixed too (Deep PILCO's estimator, DESIGN.md section 26).  With
        ``consistent=True``, ``estimator="score"`` or exploration b != 0 it is a ValueError.

        ``num_features=F`` with ``consistent=True``: the particles of ``sample_trajectories(..., consistent=True,
        num_features=F)`` and the pathwise gradient over their random-feature draws (DESIGN.md section 30), whose
        workspace does not grow with the model's centres.  With ``consistent=False``, an SMGPR model or
        ``estimator="score"`` it is a ValueError.

        -> ParticlePolicyGradient(value (float), grad [len(get_flat())], returns [num_samples]) host arrays."""
        from ..params import HostArray
        self._no_schedule("sample_policy_gradient")
        self._no_angles("sample_policy_gradient")
        self._no_noise("sample_policy_gradient")
        if estimator not in engine.ParticlePlan.ESTIMATORS:
            raise ValueError("sample_policy_gradient: estimator must be one of %s, not %r"
                             % (engine.ParticlePlan.ESTIMATORS, estimator))
        F = _feature_refusals("sample_policy_gradient", num_features, consistent, self.mgpr, estimator)
        if estimator == "score":
            self._no_mlp("sample_policy_gradient(estimator='score')")
        if consistent and estimator == "score":
            raise ValueError("sample_policy_gradient: the score-function estimator over the consistent (function-sample) "
                             "particles is engine.ConsistentGradPlan(..., estimator='score'); this method offers "
                             "estimator='pathwise' with them")
        b = float(exploration)
        _resample_refusals("sample_policy_gradient", resample, consistent, estimator, b)
        plan = self._particle_plan(m_x, s_x, n, num_samples, seed, "sample_policy_gradient", grad=True,
                                   consistent=consistent, estimator=estimator, exploration=None if b == 0.0 else b,
                                   resample=resample, num_features=F)
        g = plan.launch_grad()
        return ParticlePolicyGradient(float(g["value"].item()), self._flat_grad(g).view(HostArray),
                                      plan.ret.cpu().numpy().view(HostArray))

    def _exploration_b(self):
        """the exploration weight for the device rollout: None at b = 0, which runs the objective without it"""
        b = float(self.exploration)
        return None if b == 0.0 else b

    def _single_plan(self, m_x, s_x, n, grad=False, exploration=None):
        """RolloutPlan of one n-step rollout of the current policy from N(m_x, s_x)"""
        terms, mult_mu = self.reward_spec()
        return engine.RolloutPlan(self.mgpr.device_gp(), self.policy_spec(), terms,
                                  np.asarray(m_x, dtype=np.float64).reshape(-1), np.asarray(s_x, dtype=np.float64),
                                  int(n), R=1, mult_mu=mult_mu, grad=grad, angles=self.angle_dims,
                                  exploration=exploration, measurement_noise=self._noise_var(),
                                  schedule=self._scheduled(n))

    def predict_reward_moments(self, m_x, s_x, n):
        """Mean and variance of each step's reward along the n-step prediction from N(m_x, s_x): E[r_t] (the terms
        ``predict`` sums) and sigma_t^2 = sum_k c_k^2 Var[r_k] over the additive terms (CombinedRewards' rule), how sure
        the model is of the reward at step t (DESIGN.md section 21).  -> (mean [n], var [n]) host arrays.  A reward with
        an additive box term is a ValueError (no variance closed form)."""
        self._no_mlp("predict_reward_moments")
        from ..params import HostArray
        n = int(n)
        plan = self._single_plan(m_x, s_x, n, exploration=0.0)
        plan.forward()
        if int(plan.info[0].item()) != 0:
            raise RuntimeError("moment-matching rollout failed: covariance not positive definite")
        return (plan.step_reward[0, :n].cpu().numpy().view(HostArray),
                plan.step_var[0, :n].cpu().numpy().view(HostArray))

    def policy_gradient(self, m_x=None, s_x=None, n=None):
        """The moment-matching reward of ``predict`` (n steps from N(m_x, s_x); defaults m_init, S_init, horizon) and
        its gradient d reward / d controller.get_flat() for the current policy: the direction ``optimize_policy``
        ascends, in the layout of ``sample_policy_gradient``.  With ``exploration`` b != 0 the reward is the objective
        sum_t (E[r_t] + b sigma_t).  -> (reward (float), grad host array)."""
        self._no_mlp("policy_gradient")
        from ..params import HostArray
        m_x = self.m_init if m_x is None else m_x
        s_x = self.S_init if s_x is None else s_x
        n = self.horizon if n is None else n
        plan = self._single_plan(m_x, s_x, n, grad=True, exploration=self._exploration_b())
        plan.forward()
        g = plan.backward()
        return float(plan.reward[0].item()), self._flat_grad({k: v[0] for k, v in g.items()}).view(HostArray)

    def optimize_policy_sampled(self, maxiter=50, restarts=1, num_samples=1000, seed=None, consistent=False,
                                exploration=0.0, resample=False, num_features=None, optimizer="lbfgsb",
                                learning_rate=1e-3, betas=(0.9, 0.999), eps=1e-8, max_grad_norm=None, population=400,
                                elites=40, cem_std=0.5):
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
        needs more than half the free device memory is a ValueError naming the num_samples that would fit.

        ``exploration``: a weight b != 0 optimises PILCO's exploration objective over the particles, mean return +
        b sum_t sigma_t (``sample_policy_gradient``'s), and returns its in-sample value.  It does not read
        ``self.exploration``: pass ``exploration=self.exploration`` for the sampled counterpart of ``optimize_policy``.

        ``resample=True``: Deep PILCO's objective with its Gaussian refit at every step (``sample_policy_gradient(...,
        resample=True)``); the refit's normals are drawn once with the others.  With ``consistent=True`` or exploration
        b != 0 it is a ValueError.

        ``num_features=F`` with ``consistent=True``: the particles follow random-feature function draws (DESIGN.md
        section 30), made once as ``sample_trajectories(..., num_features=F)`` makes them; a lock-step group's workspace
        is then O(restarts num_samples horizon (D + E)) whatever the model's size.  With ``consistent=False`` or an
        SMGPR model it is a ValueError.

        ``optimizer="adam"``: stochastic gradient ascent on the expected return instead (Deep PILCO, PIPPS; DESIGN.md
        section 32).  Each of the ``maxiter`` Adam steps (``learning_rate``, ``betas``, ``eps``, the gradient's norm
        clipped to ``max_grad_norm`` when given) draws ``num_samples`` fresh particles on the device from a
        counter-based generator seeded with ``seed``, so the optimiser cannot fit the policy to one sample; the whole
        run is one CUDA graph per lock-step group replayed ``maxiter`` times.  ``consistent``, ``num_features``,
        ``resample`` and ``exploration`` mean what they mean above.  Every restart's final policy is then scored on one
        held-out sample from the same generator; the controller is set to the best, and its held-out value is returned
        (an out-of-sample estimate).  ``adam_trace`` keeps each step's in-sample values [maxiter, restarts] and whether
        each restart stepped (a restart whose value or gradient is not finite keeps its parameters).  The refusals
        above apply, and so do ValueErrors for maxiter < 1 and hyper-parameters out of range (learning_rate finite and
        > 0, betas in [0, 1), eps > 0, max_grad_norm >= 0), all raised before any device work.  The default
        optimizer ignores the four Adam arguments.

        ``optimizer="cem"``: the cross-entropy method over the flat policy vector on the same in-sample objective,
        every iteration on the device (``policy_opt.CemPolicySearch``, DESIGN.md section 33).  ``maxiter`` is its
        iteration count; each iteration rolls out ``population`` candidate policies over the fixed particles and
        refits a diagonal Gaussian to the ``elites`` best.  The search starts at the controller's current vector with
        std ``cem_std`` (a scalar or one value per parameter, finite and > 0); ``restarts`` must be 1 (the population
        is the search).  The seeded generator draws x0 and the step normals exactly as the default optimizer does (the
        same particles for the same seed), then the measurement noise's normals; the candidates' normals come from the
        counter-based generator under the same seed.  Only forward values are needed, so box terms, SafePILCO's risk
        channel, ``consistent``, and with linear and RBF controllers ``angle_dims`` and ``measurement_noise`` all work.
        The controller is set to the best candidate, whose in-sample value is returned (biased upwards, as the default
        optimizer's), and ``cem_search`` keeps the search (``trace`` [maxiter, 2] of each iteration's top value and
        elites' mean value, ``best_value``, ``mean``, ``std``).  A TimeVaryingLinearController (use ``plan``), an
        MlpController with angles or measurement noise, exploration b != 0, ``resample``, ``num_features``, restarts
        != 1, population outside 1 .. 8192, elites outside 1 .. population, maxiter < 1 or a bad ``cem_std`` is a
        ValueError raised before any device work."""
        from functools import partial
        from .. import policy_opt
        if optimizer == "cem":
            return self._optimize_policy_cem(maxiter, restarts, num_samples, seed, consistent, exploration, resample,
                                             num_features, population, elites, cem_std)
        if optimizer not in ("lbfgsb", "adam"):
            raise ValueError("optimize_policy_sampled: optimizer must be 'lbfgsb', 'adam' or 'cem', not %r"
                             % (optimizer,))
        self._no_schedule("optimize_policy_sampled")
        self._no_angles("optimize_policy_sampled")
        self._no_noise("optimize_policy_sampled")
        if int(num_samples) < 1:
            raise ValueError("optimize_policy_sampled: needs num_samples >= 1 (num_samples=%d)" % int(num_samples))
        b = float(exploration)
        _resample_refusals("optimize_policy_sampled", resample, consistent, "pathwise", b)
        F = _feature_refusals("optimize_policy_sampled", num_features, consistent, self.mgpr)
        if resample and int(num_samples) < 2:
            raise ValueError("optimize_policy_sampled: resample=True needs num_samples >= 2 (num_samples=%d)"
                             % int(num_samples))
        if not np.isfinite(b) or (b != 0.0 and int(num_samples) < 2):
            raise ValueError("optimize_policy_sampled: exploration needs a finite b and num_samples >= 2 (b=%r, "
                             "num_samples=%d)" % (exploration, int(num_samples)))
        terms, _ = self.reward_spec()
        if any(t["kind"] == _lib.REWARD_BOX for t in terms):
            raise ValueError("optimize_policy_sampled: the reward has box (risk) terms, which carry no pathwise "
                             "gradient; use optimize_policy")
        restarts = max(int(restarts), 1)
        if optimizer == "adam":
            if int(maxiter) < 1:
                raise ValueError("optimize_policy_sampled: optimizer='adam' needs maxiter >= 1 (maxiter=%d)"
                                 % int(maxiter))
            engine.adam_hyperparameters(learning_rate, betas, eps, max_grad_norm)
            return self._optimize_policy_adam(maxiter, restarts, num_samples, seed, consistent, b, resample, F,
                                              learning_rate, betas, eps, max_grad_norm)
        mgpr_trainable = self.mgpr.trainable_parameters
        for p in mgpr_trainable:
            set_trainable(p, False)
        try:
            flats0 = policy_opt.initial_flats(self.controller, restarts)
            draws = None
            if F is not None:
                x0, draws = self._feature_inputs(self.m_init, self.S_init, self.horizon, num_samples, seed, F,
                                                 "optimize_policy_sampled")
                eps, xi = None, None
            else:
                inputs = self._particle_inputs(self.m_init, self.S_init, self.horizon, num_samples, seed,
                                               "optimize_policy_sampled", resample)
                x0, eps, xi = inputs if resample else inputs + (None,)
            best_flat, best_value, _ = policy_opt.optimize(
                self, maxiter=maxiter, restarts=restarts, flats0=flats0,
                evaluator=partial(policy_opt.ParticleEvaluator, x0=x0, eps=eps, consistent=consistent,
                                  exploration=None if b == 0.0 else b, resample=resample, xi=xi, features=draws))
            self.controller.set_flat(best_flat)
        finally:
            for p in mgpr_trainable:
                set_trainable(p, True)
        return best_value

    def _optimize_policy_adam(self, maxiter, restarts, num_samples, seed, consistent, b, resample, F, learning_rate,
                              betas, eps, max_grad_norm):
        """optimize_policy_sampled(optimizer="adam") after its refusals"""
        from .. import policy_opt
        mgpr_trainable = self.mgpr.trainable_parameters
        for p in mgpr_trainable:
            set_trainable(p, False)
        try:
            flats0 = policy_opt.initial_flats(self.controller, restarts)
            if seed is None:
                seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
            best_flat, best_value, _, trace, ok = policy_opt.optimize_stochastic(
                self, int(maxiter), restarts, int(num_samples), int(seed), consistent=consistent,
                exploration=None if b == 0.0 else b, resample=resample, num_features=F, lr=learning_rate, betas=betas,
                eps=eps, max_norm=max_grad_norm, flats0=flats0)
            self.controller.set_flat(best_flat)
        finally:
            for p in mgpr_trainable:
                set_trainable(p, True)
        from ..params import HostArray
        self.adam_trace = AdamTrace(trace.view(HostArray), ok)
        return best_value

    def _optimize_policy_cem(self, maxiter, restarts, num_samples, seed, consistent, exploration, resample,
                             num_features, population, elites, cem_std):
        """optimize_policy_sampled(optimizer="cem"): every refusal before any device work, then one
        policy_opt.CemPolicySearch"""
        import torch
        from .. import policy_opt
        what = "optimize_policy_sampled(optimizer='cem')"
        c = self.controller
        if isinstance(c, controllers.TimeVaryingLinearController):
            raise ValueError("%s: a TimeVaryingLinearController plans with plan(optimizer='cem')" % what)
        if isinstance(c, controllers.MlpController):
            for on, feat in ((bool(self.angle_dims), "angles"), (self.measurement_noise is not None,
                                                                 "measurement_noise")):
                if on:
                    raise ValueError("%s: an MLP policy does not combine with %s" % (what, feat))
        for on, feat in ((float(exploration) != 0.0, "exploration (CEM's objective is the mean return)"),
                         (bool(resample), "resample=True"), (num_features is not None, "num_features")):
            if on:
                raise ValueError("%s: does not combine with %s" % (what, feat))
        if int(restarts) != 1:
            raise ValueError("%s: takes restarts=1 (the population is the search), got %d" % (what, int(restarts)))
        K, ke, iters, S, H = int(population), int(elites), int(maxiter), int(num_samples), int(self.horizon)
        if not 1 <= K <= _lib.CEM_MAX_K or not 1 <= ke <= K or iters < 1:
            raise ValueError("%s: needs 1 <= population <= %d, 1 <= elites <= population and maxiter >= 1 "
                             "(population=%d, elites=%d, maxiter=%d)" % (what, _lib.CEM_MAX_K, K, ke, iters))
        if S < 1 or H < 1:
            raise ValueError("%s: needs num_samples >= 1 and horizon >= 1 (num_samples=%d, horizon=%d)" % (what, S, H))
        n = c.get_flat().size
        std = np.asarray(cem_std, dtype=np.float64)
        if std.shape not in ((), (n,)) or not np.all(np.isfinite(std)) or not np.all(std > 0.0):
            raise ValueError("%s: cem_std must be finite and > 0, a scalar or %d values (len(get_flat())), got shape %s"
                             % (what, n, std.shape))
        noise = self._noise_var()
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        Ds = self.state_dim
        x0, g = self._start_states(self.m_init, self.S_init, S, seed)
        draw = lambda *shape: torch.randn(shape, dtype=engine.F64, device=x0.device, generator=g)
        eps = draw(S, H, Ds)                                    # _particle_inputs' step normals
        nu = draw(S, H, Ds) if noise is not None else None
        search = policy_opt.CemPolicySearch(self, K, ke, iters, S, seed, std0=std, consistent=consistent,
                                            angles=self.angle_dims, measurement_noise=noise)
        search.set_inputs(x0, eps, nu)
        best, best_value = search.run()
        c.set_flat(best.cpu().numpy())
        self.cem_search = search
        return float(best_value.item())

    def training_loss(self):
        """-(the objective optimize_policy maximises) from N(m_init, S_init) over the horizon: -predict's reward, or with
        ``exploration`` b != 0, -sum_t (E[r_t] + b sigma_t) -> [1,1] host array"""
        self._no_mlp("training_loss")
        b = self._exploration_b()
        if b is None:
            return -self.predict(self.m_init, self.S_init, self.horizon)[2]
        from ..params import HostArray
        # the taped forward, as policy_gradient runs it: the two give the same objective to the bit
        plan = self._single_plan(self.m_init, self.S_init, self.horizon, grad=True, exploration=b)
        plan.forward()
        if int(plan.info[0].item()) != 0:
            raise RuntimeError("moment-matching rollout failed: covariance not positive definite")
        return (-plan.reward[:1].reshape(1, 1)).cpu().numpy().view(HostArray)

    def compute_reward(self):
        self._no_mlp("compute_reward")
        return -self.training_loss()

    @property
    def maximum_log_likelihood_objective(self):
        return -self.training_loss()

    def compute_action(self, x_m, *, t=0):
        """pilco.py:115-116: the policy mean at a deterministic state (s = 0).  Served by a cached
        ``engine.ActionPlan`` (one captured CUDA graph per policy state) -- the per-control-step call of
        examples/utils.py:32-36.  With angle_dims, x_m is the raw state and phi(x_m) is formed on the host.
        ``t``: the step whose parameters a TimeVaryingLinearController applies (0 .. horizon-1); a stationary policy
        is the same at every step.  An MlpController: its host fp64 evaluation at the point (MlpController.compute_action)."""
        from ..params import HostArray
        c = self.controller
        if isinstance(c, controllers.MlpController):
            if self.angle_dims:
                x_m = engine.trig_feature_map(np.asarray(x_m, dtype=np.float64).reshape(1, self.state_dim),
                                              self.angle_dims)
            return c.compute_action(np.asarray(x_m, dtype=np.float64).reshape(1, -1))[0].view(HostArray)
        sched = isinstance(c, controllers.TimeVaryingLinearController)
        t = int(t) if sched else 0
        if sched and not 0 <= t < c.horizon:
            raise ValueError("compute_action: step t=%d outside the schedule's %d steps" % (t, c.horizon))
        key = (c.state_key(), t)
        if key != getattr(self, "_act_key", None):
            spec = self.policy_spec()
            if sched:                                     # step t's (W_t, b_t) as a stationary linear policy
                spec = dict(spec, W=spec["W"][t], b=spec["b"][t], schedule=False)
            self._act_plan = engine.ActionPlan(spec)
            self._act_key = key
        if self.angle_dims:
            x_m = engine.trig_feature_map(np.asarray(x_m, dtype=np.float64).reshape(1, self.state_dim), self.angle_dims)
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
        self._no_mlp("optimize_policy")
        from .. import policy_opt
        self._scheduled(self.horizon)
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

    # ---- receding-horizon planning (probabilistic MPC, Kamthe & Deisenroth 2018) --------------------------------------
    def plan(self, m_x, s_x=None, maxiter=20, restarts=1, warm_start=True, num_samples=None, seed=None,
             consistent=False, optimizer="lbfgsb", population=400, elites=40):
        """One receding-horizon step with a TimeVaryingLinearController: optimise its schedule over ``horizon`` steps
        of the moment-matching cascade from N(m_x, s_x) (s_x = None or 0: a measured state), return the first action
        u_0 = compute_action(m_x, t=0) [1,U], then shift the schedule one step (theta_t <- theta_{t+1}, the last step
        repeated) so that the next call starts from the rest of this plan.  Restart 0 starts from the current schedule
        (``warm_start=False``: from ``controller.randomize()``), the others from random draws, as ``optimize_policy``
        chooses, batches and shards them; the objective is ``optimize_policy``'s (with ``exploration``).  m_init and
        S_init are not touched.  A stationary controller is a TypeError.

        ``num_samples=S``: optimise the schedule on the in-sample mean return of S particle rollouts of the learnt
        dynamics instead (PETS-style trajectory sampling; DESIGN.md section 28), as ``optimize_policy_sampled`` does
        for a stationary policy: x0 ~ N(m_x, s_x) (every particle at m_x when s_x is None) and the step normals are
        drawn once from one generator seeded with ``seed`` and held fixed, so the objective is deterministic.
        ``consistent=True``: each particle follows one function drawn from the dynamics posterior.  Restarts, warm
        start and the shift are as above; ``exploration`` is not read.  Box terms, ``angle_dims`` and
        ``measurement_noise`` are a ValueError raised before any device work.

        ``optimizer="cem"`` (with ``num_samples``, ``restarts=1``): the cross-entropy method over the schedule's b on
        the same sampled return, every iteration on the device (``engine.CemPlan``, DESIGN.md section 31), as PETS
        plans.  ``maxiter`` is its iteration count; each iteration rolls out ``population`` candidate schedules and
        refits the sampling distribution to the ``elites`` best.  The candidates start from the controller's current
        schedule (W held fixed), its b clipped to [-pi/2, pi/2], with std pi/4.  The seeded generator draws x0 and the
        step normals exactly as the default optimizer does (the same particles for the same seed), then the
        measurement noise's normals, then the candidates' normals.  Nothing is differentiated, so box terms,
        SafePILCO's risk channel, ``angle_dims`` and ``measurement_noise`` all work.  The controller's b then holds the
        best candidate, and ``cem_plan`` the plan (its ``trace``, ``best_value`` and particles)."""
        from functools import partial
        from .. import policy_opt
        self._no_mlp("plan")
        c = self.controller
        if not isinstance(c, controllers.TimeVaryingLinearController):
            raise TypeError("plan: needs a TimeVaryingLinearController, the controller is a %s" % type(c).__name__)
        self._scheduled(self.horizon)
        Ds = self.state_dim
        m = np.asarray(m_x, dtype=np.float64).reshape(1, Ds)
        s = np.zeros((Ds, Ds)) if s_x is None else np.asarray(s_x, dtype=np.float64).reshape(Ds, Ds)
        if optimizer == "cem":
            return self._plan_cem(m, s, maxiter, restarts, warm_start, num_samples, seed, consistent, population,
                                  elites)
        if optimizer != "lbfgsb":
            raise ValueError("plan: optimizer must be 'lbfgsb' or 'cem', not %r" % (optimizer,))
        if num_samples is not None:
            self._no_angles("plan(num_samples=...)")
            self._no_noise("plan(num_samples=...)")
            if int(num_samples) < 1:
                raise ValueError("plan: needs num_samples >= 1 (num_samples=%d)" % int(num_samples))
            terms, _ = self.reward_spec()
            if any(t["kind"] == _lib.REWARD_BOX for t in terms):
                raise ValueError("plan(num_samples=...): the reward has box (risk) terms, which carry no pathwise "
                                 "gradient; plan with the moment-matching objective (num_samples=None)")
        if not warm_start:
            c.randomize()
        mgpr_trainable = self.mgpr.trainable_parameters
        for p in mgpr_trainable:
            set_trainable(p, False)
        try:
            if num_samples is None:
                evaluator = partial(policy_opt.PolicyEvaluator, m0=m, S0=s)
            else:
                x0, eps = self._particle_inputs(m, s, self.horizon, num_samples, seed, "plan")
                evaluator = partial(policy_opt.ParticleEvaluator, x0=x0, eps=eps, consistent=consistent)
            best_flat, _, _ = policy_opt.optimize(self, maxiter=maxiter, restarts=restarts, evaluator=evaluator)
            c.set_flat(best_flat)
        finally:
            for p in mgpr_trainable:
                set_trainable(p, True)
        u = self.compute_action(m, t=0)
        c.shift()
        return u

    def _plan_cem(self, m, s, maxiter, restarts, warm_start, num_samples, seed, consistent, population, elites):
        """plan(optimizer="cem"): every refusal before any device work, then one engine.CemPlan"""
        import torch
        if num_samples is None or int(num_samples) < 1:
            raise ValueError("plan(optimizer='cem'): needs num_samples >= 1 (num_samples=%r)" % (num_samples,))
        if int(restarts) != 1:
            raise ValueError("plan(optimizer='cem'): takes restarts=1 (the population is the search), got %d"
                             % int(restarts))
        K, ke, iters = int(population), int(elites), int(maxiter)
        if not 1 <= K <= _lib.CEM_MAX_K or not 1 <= ke <= K or iters < 1:
            raise ValueError("plan(optimizer='cem'): needs 1 <= population <= %d, 1 <= elites <= population and "
                             "maxiter >= 1 (population=%d, elites=%d, maxiter=%d)" % (_lib.CEM_MAX_K, K, ke, iters))
        c, H, S, U, Ds = self.controller, int(self.horizon), int(num_samples), self.control_dim, self.state_dim
        if H < 1:
            raise ValueError("plan(optimizer='cem'): needs horizon >= 1")
        if not warm_start:
            c.randomize()
        spec = c.policy_spec()
        spec["b"] = np.clip(spec["b"], -engine.CEM_BOUND, engine.CEM_BOUND)
        terms, mult_mu = self.reward_spec()
        noise = self._noise_var()
        x0, g = self._start_states(m, s, S, seed)
        draw = lambda *shape: torch.randn(shape, dtype=engine.F64, device=x0.device, generator=g)
        eps = draw(S, H, Ds)                                    # _particle_inputs' step normals
        nu = draw(S, H, Ds) if noise is not None else None
        xi = draw(iters, K, H, U)
        plan = engine.CemPlan(self.mgpr.device_gp(), spec, terms, S, H, K, ke, iters, mult_mu=mult_mu,
                              consistent=consistent, angles=self.angle_dims, measurement_noise=noise)
        plan.set_inputs(x0, eps, xi, nu=nu)
        plan.launch()
        b = np.array(c.b, dtype=np.float64)
        b[:H] = plan.best_b.cpu().numpy()
        c.b.assign(b)
        self.cem_plan = plan
        u = self.compute_action(m, t=0)
        c.shift()
        return u
