"""MGPR -- E independent SE-ARD GPs sharing their inputs, predicted at a Gaussian input by moment
matching on the device (drop-in for the reference class at pilco/models/mgpr.py:17-190).

Host side (this file): parameter objects, data handling, training driver.
Device side: ``pilco_gp_factorize`` (mgpr.py:81-89) and ``pilco_mm_forward`` (mgpr.py:91-149) through
``pilco_b200.engine``.  Factorisations are cached per (data, hyper-parameter) state instead of being
recomputed on every call as the reference does (mgpr.py:77-79).
"""
import numbers

import numpy as np
import torch

from .. import engine, gp_training
from ..params import Parameter, Softplus, host


class Kernel:
    """SE-ARD kernel parameter holder (gpflow.kernels.SquaredExponential surface)."""

    def __init__(self, D, lengthscale_lower=0.0):
        self.lengthscales = Parameter(np.ones(D), transform=Softplus(lengthscale_lower), name="lengthscales")
        self.variance = Parameter(1.0, transform=Softplus(0.0), name="variance")

    def K(self, X1, X2=None):
        X1 = np.asarray(X1, dtype=np.float64)
        X2 = X1 if X2 is None else np.asarray(X2, dtype=np.float64)
        ell = np.asarray(self.lengthscales)
        a, b = X1 / ell, X2 / ell
        d2 = (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * a @ b.T
        return float(self.variance) * np.exp(-0.5 * np.maximum(d2, 0.0))


class Likelihood:
    def __init__(self, variance=1.0):
        self.variance = Parameter(variance, transform=Softplus(1e-6), name="likelihood_variance")
        self.prior = None


class GPRModel:
    """One output GP: kernel + Gaussian likelihood + its (X, y) data (gpflow.models.GPR surface)."""

    def __init__(self, data, kernel):
        self.data = (np.asarray(data[0], dtype=np.float64), np.asarray(data[1], dtype=np.float64))
        self.kernel = kernel
        self.likelihood = Likelihood(1.0)

    @property
    def parameters(self):
        return [self.kernel.lengthscales, self.kernel.variance, self.likelihood.variance]

    @property
    def trainable_parameters(self):
        return [p for p in self.parameters if p.trainable]

    def _loss(self, vals):
        X = torch.as_tensor(np.asarray(self.data[0]), dtype=torch.float64)
        y = torch.as_tensor(np.asarray(self.data[1]), dtype=torch.float64)[:, 0]
        ell, sf2, sn2 = vals
        return gp_training.gpr_loss(X, y, ell, sf2, sn2,
                                    ell_prior=self.kernel.lengthscales.prior, sf2_prior=self.kernel.variance.prior)

    def training_loss(self):
        return float(self._loss([torch.as_tensor(p.value(), dtype=torch.float64) for p in self.parameters]))

    def optimize(self, maxiter=None):
        return gp_training.minimize(self._loss, self.parameters, maxiter=maxiter)

    # ---- prediction at deterministic inputs (gpflow.models.GPR.predict_f / predict_y / predict_log_density) -----------
    _owner = None           # (MGPR, output index) of the models an MGPR creates

    def _hypers(self):
        return (np.asarray(self.kernel.lengthscales, dtype=np.float64).reshape(1, -1),
                np.asarray(self.kernel.variance, dtype=np.float64).reshape(1),
                np.asarray(self.likelihood.variance, dtype=np.float64).reshape(1))

    def _own_key(self):
        parts = [np.asarray(self.data[0], dtype=np.float64), np.asarray(self.data[1], dtype=np.float64), *self._hypers()]
        return hash(tuple(np.ascontiguousarray(p).tobytes() for p in parts))

    def _own_factorize(self):
        ell, sf2, sn2 = self._hypers()
        return engine.gp_factorize(np.asarray(self.data[0]), np.asarray(self.data[1]).reshape(-1, 1), ell, sf2, sn2)

    def _predict_source(self):
        """(DeviceGP, output index) holding this model's posterior.  A model of an MGPR whose inputs are the MGPR's
        uses the MGPR's resident factorisation (the one the rollout uses, appended rows included); any other model
        factorises its own data, cached until data or hyper-parameters change."""
        engine.device()
        if self._owner is not None:
            mgpr, i = self._owner
            if mgpr.mm_mode == 0 and i < len(mgpr.models) and mgpr.models[i] is self:
                try:
                    same = np.array_equal(np.asarray(self.data[0], dtype=np.float64), mgpr.X) and mgpr.Y.shape[1] == len(mgpr.models)
                except ValueError:                  # outputs with different row counts: no common factorisation
                    same = False
                if same:
                    return mgpr.device_gp(), i
        return self._own_device_gp(), 0

    def _own_device_gp(self):
        key = self._own_key()
        cached = getattr(self, "_own_gp", None)
        if cached is None or cached[0] != key:
            gp = self._own_factorize()
            if int(gp.info.max().item()):
                raise RuntimeError("Cholesky decomposition was not successful (matrix not positive definite)")
            self._own_gp = (key, gp)
        return self._own_gp[1]

    def _predict_device(self, Xnew, full_cov, full_output_cov):
        if full_output_cov:
            raise NotImplementedError("full_output_cov: a GPRModel has a single output")
        gp, e = self._predict_source()
        return engine.gp_predict(gp, Xnew, e0=e, ne=1, full_cov=full_cov)

    def predict_f(self, Xnew, full_cov=False, full_output_cov=False):
        """Latent posterior at Xnew [T,D]: mean [T,1] and variance [T,1] ([1,T,T] with ``full_cov``)."""
        mean, var = self._predict_device(Xnew, full_cov, full_output_cov)
        return host(mean), host(var)

    def predict_y(self, Xnew, full_cov=False, full_output_cov=False):
        """Predictive of the observations: predict_f's mean and variance + the likelihood variance."""
        if full_cov:
            raise NotImplementedError("predict_y with full_cov=True: add the likelihood variance to predict_f's diagonal")
        mean, var = self._predict_device(Xnew, False, full_output_cov)
        return host(mean), host(var + float(self.likelihood.variance))

    def predict_f_samples(self, Xnew, num_samples=None, full_cov=True, full_output_cov=False, *, seed=None):
        """Latent functions drawn from the posterior at Xnew [T,D]: [num_samples,T,1] ([T,1] when num_samples is None).
        ``full_cov=True`` draws mean + L eps with L = chol(cov + 1e-6 I), the correlated function values at the T
        points; ``full_cov=False`` draws each point from its own marginal.  The standard normals come from one device
        ``torch.Generator`` seeded with ``seed`` (from ``np.random`` when None): the same seed gives the same draw."""
        if num_samples is not None and (isinstance(num_samples, bool) or not isinstance(num_samples, numbers.Integral)
                                        or num_samples < 1):
            raise ValueError("predict_f_samples: num_samples must be None or an integer >= 1, got %r" % (num_samples,))
        if full_output_cov:
            raise NotImplementedError("full_output_cov: a GPRModel has a single output")
        gp, e = self._predict_source()
        Xs = engine.dev(Xnew)
        S = 1 if num_samples is None else int(num_samples)
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        g = torch.Generator(device=Xs.device)
        g.manual_seed(int(seed))
        eps = torch.randn((S, Xs.shape[0], 1), dtype=engine.F64, device=Xs.device, generator=g)
        samples, info = engine.gp_predict_samples(gp, Xs, eps, e0=e, ne=1, full_cov=full_cov)
        if int(info.max().item()):
            raise RuntimeError("Cholesky decomposition was not successful (posterior covariance + jitter not positive "
                               "definite)")
        return host(samples[0] if num_samples is None else samples)

    def predict_log_density(self, data, full_cov=False, full_output_cov=False):
        """log N(Y | mean, var_f + sn2) at each row of data = (X [T,D], Y [T,1]) -> [T]."""
        if full_cov:
            raise NotImplementedError("predict_log_density with full_cov=True")
        mean, var = self._predict_device(data[0], False, full_output_cov)
        Y = engine.dev(data[1]).reshape(mean.shape)
        vy = var + float(self.likelihood.variance)
        return host((-0.5 * (np.log(2.0 * np.pi) + torch.log(vy) + (Y - mean) ** 2 / vy)).sum(-1))


def randomize(model, mean=1, sigma=0.01):
    """pilco/models/mgpr.py:8-15"""
    model.kernel.lengthscales.assign(mean + sigma * np.random.normal(size=model.kernel.lengthscales.shape))
    model.kernel.variance.assign(mean + sigma * np.random.normal(size=model.kernel.variance.shape))
    if model.likelihood.variance.trainable:
        model.likelihood.variance.assign(mean + sigma * np.random.normal())


class MGPR:
    mm_mode = 0         # 0: GP with trace term; 1: deterministic GP (RbfController)

    def __init__(self, data, name=None):
        self.name = name
        self.num_outputs = data[1].shape[1]
        self.num_dims = data[0].shape[1]
        self.num_datapoints = data[0].shape[0]
        self.create_models(data)
        self.optimizers = []
        self._cache_key = None
        self._cache_gp = None

    # ---- construction / data (mgpr.py:28-45) -------------------------------------------------
    def create_models(self, data):
        self.models = []
        for i in range(self.num_outputs):
            kern = Kernel(data[0].shape[1])
            kern.lengthscales.prior = (1.1, 1.0 / 10.0)        # Gamma(alpha, rate)   mgpr.py:33
            kern.variance.prior = (1.5, 1.0 / 2.0)             # mgpr.py:34
            self.models.append(GPRModel((data[0], data[1][:, i:i + 1]), kern))
            self.models[-1]._owner = (self, i)              # predict_f uses this MGPR's factorisation

    def set_data(self, data):
        """``data`` = (X, Y) in the models' input layout.  A PILCO with angle_dims trains its models on [phi(x), u]
        (set by PILCO as ``_input_width``): raw [x, u] data of another width is a ValueError naming PILCO.set_data."""
        w = getattr(self, "_input_width", None)
        if w is not None and np.asarray(data[0]).shape[1] != w:
            raise ValueError("these models take inputs [phi(x), u] of width %d, got width %d: pass raw (X = [x, u], Y) "
                             "data to PILCO.set_data, which applies phi" % (w, np.asarray(data[0]).shape[1]))
        for i, model in enumerate(self.models):
            if isinstance(model.data[0], Parameter):
                model.X.assign(data[0])
                model.Y.assign(data[1][:, i:i + 1])
                model.data = [model.X, model.Y]
            else:
                model.data = (np.asarray(data[0], dtype=np.float64), np.asarray(data[1][:, i:i + 1], dtype=np.float64))
        self.num_datapoints = np.asarray(data[0]).shape[0]

    # ---- training (mgpr.py:47-75) -----------------------------------------------------------------
    def optimize(self, restarts=1, maxiter=None):
        """All outputs and restarts in lock step on the device (pilco_gp_nlml; gp_device_training.py)."""
        from .. import gp_device_training
        self.optimizers = [True] * len(self.models)
        return gp_device_training.optimize_mgpr(self, restarts=restarts, maxiter=maxiter)

    def optimize_host(self, restarts=1, maxiter=None):
        """Host path (torch-CPU autograd + SciPy): used by SMGPR (FITC objective, gp_training.py)."""
        for model in self.models:
            model.optimize(maxiter)
        self.optimizers = [True] * len(self.models)
        for model in self.models:
            best = [p.value() for p in model.parameters]
            best_loss = model.training_loss()
            for _ in range(restarts):
                randomize(model)
                model.optimize(maxiter)
                loss = model.training_loss()
                if loss < best_loss:          # the reference's bookkeeping keeps the last restart
                    best_loss = loss          # (mgpr.py:58-75); keeping the best is the documented intent
                    best = [p.value() for p in model.parameters]
            for p, v in zip(model.parameters, best):
                p.assign(v)

    @property
    def trainable_parameters(self):
        return [p for m in self.models for p in m.trainable_parameters]

    @property
    def parameters(self):
        return [p for m in self.models for p in m.parameters]

    # ---- stacked views (mgpr.py:151-190) -------------------------------------------------------
    @property
    def X(self):
        return np.asarray(self.models[0].data[0], dtype=np.float64)

    @property
    def Y(self):
        return np.concatenate([np.asarray(m.data[1], dtype=np.float64) for m in self.models], axis=1)

    @property
    def data(self):
        return (self.X, self.Y)

    @property
    def lengthscales(self):
        return np.stack([np.asarray(m.kernel.lengthscales) for m in self.models])

    @property
    def variance(self):
        return np.stack([np.asarray(m.kernel.variance) for m in self.models]).reshape(-1)

    @property
    def noise(self):
        return np.stack([np.asarray(m.likelihood.variance) for m in self.models]).reshape(-1)

    def centralized_input(self, m):
        return self.centres - np.asarray(m)

    @property
    def centres(self):
        return self.X

    def K(self, X1, X2=None):
        return np.stack([m.kernel.K(X1, X2) for m in self.models])

    # ---- device path ---------------------------------------------------------------------------
    def _state_key(self):
        parts = [self.X, self.Y, self.lengthscales, self.variance, self.noise]
        return hash(tuple(np.ascontiguousarray(p).tobytes() for p in parts))

    def _factorize(self):
        return engine.gp_factorize(self.X, self.Y, self.lengthscales, self.variance, self.noise,
                                   need_iK=(self.mm_mode == 0), mode=self.mm_mode)

    # incremental set_data (SURVEY section 8f-2): rows appended + hyper-parameters unchanged -> O(n^2 k) update of the
    # resident triangular inverse instead of a new O(n^3) factorisation.  After MAX_APPENDS consecutive appends or when
    # more rows arrive than the model holds, it is refactorised from scratch.  The round-off of the appends grows
    # slowly: on PILCO-like episodes at the noise floor (sn2 = 1e-6) eight appends of 40 rows leave iK and beta within
    # 9 and 16 eps of their condition scales (tests/test_gpu_fact_regimes.py), where a refactorisation stays within 2.
    MAX_APPENDS = 8
    incremental = True

    def _hyper_key(self):
        return hash(tuple(np.ascontiguousarray(p).tobytes() for p in (self.lengthscales, self.variance, self.noise)))

    def _try_append(self):
        """The cached model extended by the appended rows, or None when this is not a pure append."""
        gp, snap = self._cache_gp, getattr(self, "_cache_snap", None)
        if not self.incremental or gp is None or snap is None or type(self)._factorize is not MGPR._factorize:
            return None
        X, Y = self.X, self.Y
        X0, Y0, hk = snap
        n0, n1 = X0.shape[0], X.shape[0]
        if not (n0 < n1 <= 2 * n0) or X.shape[1] != X0.shape[1] or Y.shape[1] != Y0.shape[1] or hk != self._hyper_key():
            return None
        if getattr(gp, "appends", 0) >= self.MAX_APPENDS:
            return None
        if not (np.array_equal(X[:n0], X0) and np.array_equal(Y[:n0], Y0)):
            return None
        new = engine.gp_append(gp, X, Y)
        return new if int(new.info.max().item()) == 0 else None

    def device_gp(self):
        """Factorised device model, resident until data or hyper-parameters change; appended rows update it in
        place of a refactorisation (``_try_append``)."""
        key = self._state_key()
        if key != self._cache_key:
            gp = self._try_append() if self.mm_mode == 0 else None
            self.last_update = "append" if gp is not None else "factorize"
            if gp is None:
                gp = self._factorize()
                bad = int(gp.info.max().item())
                if bad:
                    raise RuntimeError("Cholesky decomposition was not successful (Gram matrix not positive definite)")
            self._cache_gp, self._cache_key = gp, key
            self._cache_snap = (self.X.copy(), self.Y.copy(), self._hyper_key())
        return self._cache_gp

    def calculate_factorizations(self):
        """(iK [E,n,n], beta [E,n]) as CUDA tensors  (mgpr.py:81-89)."""
        gp = self.device_gp()
        iK = gp.iK[:, :gp.n, :gp.n] if gp.iK is not None else None
        self._last_fact = (iK, gp.beta, self._cache_key)
        return iK, gp.beta

    def _gp_from_factors(self, iK, beta):
        """Temporary device model around caller-supplied factors (any array-like [E,n,n] / [E,n]): the reference's
        predict_given_factorizations computes with whatever it is handed (mgpr.py:91-149; RbfController passes
        ``0.0 * iK``, controllers.py:116), so custom / modified factors must drive the result here too."""
        base = self.device_gp()
        n, E = base.n, base.E
        beta_d = engine.dev(beta.detach() if isinstance(beta, torch.Tensor) else beta).reshape(E, n)
        iK_d = engine.dev(iK.detach() if isinstance(iK, torch.Tensor) else iK).reshape(E, n, n)
        ldk = engine.pad_n(n)
        pad = torch.zeros((E, ldk, ldk), dtype=torch.float64, device=iK_d.device)
        pad[:, :n, :n] = iK_d
        return engine.DeviceGP(base.X, base.ell, base.sf2, beta_d, pad, ldk, mode=0)

    def predict_given_factorizations(self, m, s, iK=None, beta=None):
        """mgpr.py:91-149 on the device.  With no factors, or with exactly the objects ``calculate_factorizations``
        returned for the current state, the cached device model is used; any other ``iK`` / ``beta`` is honoured
        (a temporary device model is built from them) -- never silently ignored."""
        gp = self.device_gp()
        last = getattr(self, "_last_fact", None)
        own = last is not None and last[2] == self._cache_key and iK is last[0] and beta is last[1]
        if (iK is None) != (beta is None):
            raise ValueError("predict_given_factorizations: pass both iK and beta (or neither)")
        if iK is not None and not own:
            gp = self._gp_from_factors(iK, beta)
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        s = np.asarray(s, dtype=np.float64).reshape(1, gp.D, gp.D)
        M, S, V, info = engine.mm_forward(gp, m, s)
        if int(info[0].item()):
            raise RuntimeError("moment matching failed: input covariance system not positive definite")
        return host(M), host(S[0]), host(V[0])

    def predict_on_noisy_inputs(self, m, s):
        """mgpr.py:77-79 -> (M [1,E], S [E,E], V [D,E])"""
        return self.predict_given_factorizations(m, s)
