"""Policies (drop-in for pilco/controllers.py): ``squash_sin``, ``LinearController``, ``RbfController``, the
step-indexed ``TimeVaryingLinearController`` of receding-horizon planning (``PILCO.plan``), and the tanh
``MlpController`` that the particle rollouts train (``PILCO.optimize_policy_sampled``).
All moment computations run on the device through the C ABI (``pilco_squash_sin``,
``pilco_linear_action``, ``pilco_gp_factorize`` + ``pilco_mm_forward`` in deterministic-GP mode)."""
import numpy as np

from . import engine, _lib
from .models.mgpr import MGPR, Kernel
from .params import HostArray, Parameter, Softplus, host, set_trainable


def _max_action_vec(max_action, k):
    if max_action is None:
        return np.ones(k)
    return np.broadcast_to(np.asarray(max_action, dtype=np.float64).reshape(-1), (k,)).copy()


def squash_sin(m, s, max_action=None):
    """Moments of max_action*sin(x), x~N(m,s) (controllers.py:13-36; gSin.m).  m [1,k], s [k,k]."""
    m = np.asarray(m, dtype=np.float64).reshape(1, -1)
    k = m.shape[1]
    s = np.asarray(s, dtype=np.float64).reshape(1, k, k)
    M, S, C = engine.squash_sin(m, s, _max_action_vec(max_action, k))
    return host(M), host(S[0]), host(C[0])


class LinearController:
    """u = W x + b (controllers.py:39-63)."""

    def __init__(self, state_dim, control_dim, max_action=1.0):
        self.W = Parameter(np.random.rand(control_dim, state_dim), name="W")
        self.b = Parameter(np.random.rand(1, control_dim), name="b")
        self.max_action = max_action

    @property
    def parameters(self):
        return [self.W, self.b]

    @property
    def trainable_parameters(self):
        return [p for p in self.parameters if p.trainable]

    def compute_action(self, m, s, squash=True):
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        Ds = m.shape[1]
        s = np.asarray(s, dtype=np.float64).reshape(1, Ds, Ds)
        U = self.W.shape[0]
        M, S, V = engine.linear_action(np.asarray(self.W), np.asarray(self.b).reshape(U), m, s)
        if squash:
            M, S, C = engine.squash_sin(M, S, _max_action_vec(self.max_action, U))
            V = V @ C
        return host(M), host(S[0]), host(V[0])

    def randomize(self):
        mean, sigma = 0, 1
        self.W.assign(mean + sigma * np.random.normal(size=self.W.shape))
        self.b.assign(mean + sigma * np.random.normal(size=self.b.shape))

    # ---- flat parameter vector for the batched policy optimiser ---------------------------------
    def policy_spec(self, flat=None):
        U, Ds = self.W.shape
        if flat is None:
            W, b = np.asarray(self.W), np.asarray(self.b).reshape(U)
        else:
            flat = np.asarray(flat, dtype=np.float64)
            W = flat[..., :U * Ds].reshape(flat.shape[:-1] + (U, Ds))
            b = flat[..., U * Ds:].reshape(flat.shape[:-1] + (U,))
        return dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=_max_action_vec(self.max_action, U),
                    W=W, b=b)

    def state_key(self):
        return hash((np.asarray(self.W).tobytes(), np.asarray(self.b).tobytes(),
                     np.asarray(self.max_action, dtype=np.float64).tobytes()))

    def get_flat(self):
        return np.concatenate([np.asarray(self.W).ravel(), np.asarray(self.b).ravel()])

    def set_flat(self, flat):
        U, Ds = self.W.shape
        self.W.assign(np.asarray(flat[:U * Ds]).reshape(U, Ds))
        self.b.assign(np.asarray(flat[U * Ds:]).reshape(1, U))


class TimeVaryingLinearController:
    """u_t = W_t x + b_t, one (W_t, b_t) per step t = 0 .. horizon-1 (squashed by squash_sin in the rollout): the
    action sequences that probabilistic MPC plans through the moment-matching cascade (Kamthe & Deisenroth 2018;
    DESIGN.md section 27).  ``feedback=False`` is the open-loop sequence u_t = b_t: W stays 0 and is not trainable.
    The flat vector is [W (horizon*U*Ds) | b (horizon*U)], or [b] without feedback, step-major."""

    def __init__(self, state_dim, control_dim, horizon, max_action=1.0, feedback=True):
        if int(horizon) < 1:
            raise ValueError("TimeVaryingLinearController: horizon must be >= 1, got %r" % horizon)
        self.horizon, self.feedback = int(horizon), bool(feedback)
        H, U, Ds = self.horizon, int(control_dim), int(state_dim)
        W0 = 0.1 * np.random.randn(H, U, Ds) if self.feedback else np.zeros((H, U, Ds))
        self.W = Parameter(W0, trainable=self.feedback, name="W")
        self.b = Parameter(0.1 * np.random.randn(H, U), name="b")
        self.max_action = max_action

    @property
    def parameters(self):
        return [self.W, self.b]

    @property
    def trainable_parameters(self):
        return [p for p in self.parameters if p.trainable]

    def compute_action(self, m, s, squash=True, t=0):
        """the moments of step t's action at N(m, s) -> (M [1,U], S [U,U], V [Ds,U])"""
        t = int(t)
        if not 0 <= t < self.horizon:
            raise ValueError("compute_action: step t=%d outside the schedule's %d steps" % (t, self.horizon))
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        Ds = m.shape[1]
        s = np.asarray(s, dtype=np.float64).reshape(1, Ds, Ds)
        U = self.b.shape[1]
        M, S, V = engine.linear_action(np.asarray(self.W)[t], np.asarray(self.b)[t], m, s)
        if squash:
            M, S, C = engine.squash_sin(M, S, _max_action_vec(self.max_action, U))
            V = V @ C
        return host(M), host(S[0]), host(V[0])

    def randomize(self):
        """small random parameters around 0: b ~ N(0, 0.1^2) (and W likewise with feedback)"""
        if self.feedback:
            self.W.assign(0.1 * np.random.normal(size=self.W.shape))
        self.b.assign(0.1 * np.random.normal(size=self.b.shape))

    def shift(self):
        """the receding horizon's warm start: theta_t <- theta_{t+1}, the last step repeated"""
        for p in self.parameters:
            v = np.asarray(p)
            p.assign(np.concatenate([v[1:], v[-1:]]))

    def policy_spec(self, flat=None):
        """the scheduled spec of engine.RolloutPlan(..., schedule=True): W [lead.., H, U, Ds], b [lead.., H, U]"""
        H, U, Ds = self.W.shape
        if flat is None:
            W, b = np.asarray(self.W), np.asarray(self.b)
        else:
            flat = np.asarray(flat, dtype=np.float64)
            lead = flat.shape[:-1]
            nW = H * U * Ds if self.feedback else 0
            W = flat[..., :nW].reshape(lead + (H, U, Ds)) if nW else np.zeros(lead + (H, U, Ds))
            b = flat[..., nW:].reshape(lead + (H, U))
        return dict(kind=_lib.POLICY_LINEAR, Ds=Ds, U=U, squash=True, max_action=_max_action_vec(self.max_action, U),
                    W=W, b=b, schedule=True)

    def state_key(self):
        return hash((np.asarray(self.W).tobytes(), np.asarray(self.b).tobytes(),
                     np.asarray(self.max_action, dtype=np.float64).tobytes()))

    def get_flat(self):
        b = np.asarray(self.b).ravel()
        return np.concatenate([np.asarray(self.W).ravel(), b]) if self.feedback else b

    def set_flat(self, flat):
        H, U, Ds = self.W.shape
        flat = np.asarray(flat, dtype=np.float64)
        nW = H * U * Ds if self.feedback else 0
        if nW:
            self.W.assign(flat[:nW].reshape(H, U, Ds))
        self.b.assign(flat[nW:].reshape(H, U))

    def flat_grad(self, gW, gb):
        """per-step cotangents gW [n, U, Ds], gb [n, U] of an n-step rollout (n <= horizon) -> the get_flat() layout,
        zero for the steps the rollout does not reach"""
        H, U, Ds = self.W.shape
        n = np.shape(gb)[0]
        fb = np.zeros((H, U))
        fb[:n] = np.asarray(gb).reshape(n, U)
        if not self.feedback:
            return fb.ravel()
        fW = np.zeros((H, U, Ds))
        fW[:n] = np.asarray(gW).reshape(n, U, Ds)
        return np.concatenate([fW.ravel(), fb.ravel()])


class MlpController:
    """A tanh multilayer perceptron, the policy Deep PILCO (Gal, McAllister & Rasmussen 2016) trains on sampled returns:
    h_1 = tanh(A_1 [x; 1]), (two layers) h_2 = tanh(A_2 [h_1; 1]), z = A_out [h_L; 1], u = max_action sin(z)
    (DESIGN.md section 29).  Each A is a Parameter [out, in + 1] with the bias as its last column; ``get_flat()`` is
    the blocks in order, row-major, output layer last (the device's theta).  ``hidden``: one or two widths of 1 .. 64.

    Moment matching has no closed form for it: the particle methods of ``PILCO`` (``sample_trajectories``,
    ``sample_reward_moments``, ``sample_policy_gradient`` and ``optimize_policy_sampled``) run it, the moment-matching
    ones refuse it.  ``compute_action`` evaluates it at a point."""

    def __init__(self, state_dim, control_dim, hidden=(64, 64), max_action=1.0):
        hidden = tuple(int(w) for w in hidden)
        if len(hidden) not in (1, 2) or any(w < 1 or w > engine.MLP_MAX_WIDTH for w in hidden):
            raise ValueError("MlpController: 1 or 2 hidden layers of 1 .. %d units, got hidden=%s"
                             % (engine.MLP_MAX_WIDTH, hidden))
        self.state_dim, self.control_dim, self.hidden = int(state_dim), int(control_dim), hidden
        widths = [self.state_dim] + list(hidden) + [self.control_dim]
        self.layers = [Parameter(np.zeros((widths[l + 1], widths[l] + 1)), name="A%d" % (l + 1))
                       for l in range(len(widths) - 1)]
        self.max_action = max_action
        self.randomize()

    @property
    def parameters(self):
        return list(self.layers)

    @property
    def trainable_parameters(self):
        return [p for p in self.parameters if p.trainable]

    def randomize(self):
        """weights N(0, 1 / fan_in), biases 0, from np.random"""
        for A in self.layers:
            out, fan = A.shape[0], A.shape[1] - 1
            W = np.random.normal(size=(out, fan)) / np.sqrt(fan)
            A.assign(np.concatenate([W, np.zeros((out, 1))], axis=1))

    def get_flat(self):
        return np.concatenate([np.asarray(A.numpy()).ravel() for A in self.layers])

    def set_flat(self, flat):
        flat, o = np.asarray(flat, dtype=np.float64), 0
        for A in self.layers:
            n = int(np.prod(A.shape))
            A.assign(flat[o:o + n].reshape(A.shape))
            o += n

    def policy_spec(self, flats=None):
        """the device's spec: theta = ``flats`` ([n_theta] or [R, n_theta]) or the current parameters"""
        theta = self.get_flat() if flats is None else np.asarray(flats, dtype=np.float64)
        return dict(kind=_lib.POLICY_MLP, Ds=self.state_dim, U=self.control_dim, squash=True,
                    max_action=_max_action_vec(self.max_action, self.control_dim), hidden=self.hidden, theta=theta)

    def state_key(self):
        return hash((self.get_flat().tobytes(), np.asarray(self.max_action, dtype=np.float64).tobytes()))

    def compute_action(self, m, s=None, squash=True):
        """the action at the point m [1, Ds] (s None or 0: an MLP has no moment closed form) -> (M [1,U], S [U,U] = 0,
        V [Ds,U] = 0), the triple the other controllers return at s = 0.  A host fp64 evaluation of one point."""
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        if s is not None and np.any(np.asarray(s, dtype=np.float64) != 0.0):
            raise ValueError("MlpController.compute_action: evaluates at a point only (s = 0); propagate a state "
                             "distribution with PILCO's particle methods (sample_trajectories)")
        h = m[0]
        for l, A in enumerate(self.layers):
            A = np.asarray(A.numpy())
            h = A[:, :-1] @ h + A[:, -1]
            if l < len(self.layers) - 1:
                h = np.tanh(h)
        U = self.control_dim
        if squash:
            h = _max_action_vec(self.max_action, U) * np.sin(h)
        return (h.reshape(1, U).view(HostArray), np.zeros((U, U)).view(HostArray),
                np.zeros((m.shape[1], U)).view(HostArray))


class FakeLikelihood:
    def __init__(self, variance):
        self.variance = Parameter(variance, transform=Softplus(1e-6), trainable=False, name="likelihood_variance")


class FakeGPR:
    """Parameter holder of one policy output (controllers.py:66-78): trainable centres X (shared) and
    targets Y, fixed noise 1e-4."""

    def __init__(self, data, kernel, X=None, likelihood_variance=1e-4):
        self.X = Parameter(data[0], name="DataX") if X is None else X
        self.Y = Parameter(data[1], name="DataY")
        self.data = [self.X, self.Y]
        self.kernel = kernel
        self.likelihood = FakeLikelihood(likelihood_variance)

    @property
    def parameters(self):
        return [self.X, self.Y, self.kernel.lengthscales, self.kernel.variance, self.likelihood.variance]

    @property
    def trainable_parameters(self):
        return [p for p in self.parameters if p.trainable]


class RbfController(MGPR):
    """RBF network policy = deterministic GP (controllers.py:80-129; gp2.m)."""
    mm_mode = 1

    def __init__(self, state_dim, control_dim, num_basis_functions, max_action=1.0):
        MGPR.__init__(self, [np.random.randn(num_basis_functions, state_dim),
                             0.1 * np.random.randn(num_basis_functions, control_dim)])
        for model in self.models:
            model.kernel.variance.assign(1.0)
            set_trainable(model.kernel.variance, False)
        self.max_action = max_action

    def create_models(self, data):
        self.models = []
        for i in range(self.num_outputs):
            kernel = Kernel(data[0].shape[1], lengthscale_lower=1e-3)        # controllers.py:100
            kernel.lengthscales.prior = (1.1, 1.0 / 10.0)
            if i == 0:
                self.models.append(FakeGPR((data[0], data[1][:, i:i + 1]), kernel))
            else:
                self.models.append(FakeGPR((data[0], data[1][:, i:i + 1]), kernel, self.models[-1].X))

    def compute_action(self, m, s, squash=True):
        """controllers.py:108-121 -> (M [1,U], S [U,U], V [Ds,U])"""
        gp = self.device_gp()
        m = np.asarray(m, dtype=np.float64).reshape(1, -1)
        s = np.asarray(s, dtype=np.float64).reshape(1, gp.D, gp.D)
        M, S, V, info = engine.mm_forward(gp, m, s)      # mode 1: no trace term, +1e-6 on the diagonal
        if squash:
            M, S, C = engine.squash_sin(M, S, _max_action_vec(self.max_action, gp.E))
            V = V @ C
        return host(M), host(S[0]), host(V[0])

    def randomize(self):
        print("Randomising controller")
        for m in self.models:
            m.X.assign(np.random.normal(size=m.data[0].shape))
            m.Y.assign(self.max_action / 10 * np.random.normal(size=m.data[1].shape))
            mean, sigma = 1, 0.1
            m.kernel.lengthscales.assign(mean + sigma * np.random.normal(size=m.kernel.lengthscales.shape))

    def state_key(self):
        return hash((self._state_key(), np.asarray(self.max_action, dtype=np.float64).tobytes()))

    # ---- flat parameter vector: [centres (bf*Ds) | targets (bf*U) | unconstrained lengthscales (U*Ds)] ----
    @property
    def policy_shapes(self):
        bf, Ds = self.models[0].X.shape
        return bf, Ds, self.num_outputs

    def get_flat(self):
        X = np.asarray(self.models[0].X).ravel()
        Y = self.Y.ravel()
        th = np.concatenate([m.kernel.lengthscales.unconstrained.ravel() for m in self.models])
        return np.concatenate([X, Y, th])

    def split_flat(self, flat):
        bf, Ds, U = self.policy_shapes
        flat = np.asarray(flat, dtype=np.float64)
        lead = flat.shape[:-1]
        X = flat[..., :bf * Ds].reshape(lead + (bf, Ds))
        Y = flat[..., bf * Ds:bf * Ds + bf * U].reshape(lead + (bf, U))
        th = flat[..., bf * Ds + bf * U:].reshape(lead + (U, Ds))
        return X, Y, th

    def set_flat(self, flat):
        X, Y, th = self.split_flat(flat)
        self.models[0].X.assign(X)
        for i, m in enumerate(self.models):
            m.Y.assign(Y[:, i:i + 1])
            m.kernel.lengthscales.set_unconstrained(th[i])
