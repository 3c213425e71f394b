"""Generate tests/golden/obs_noise.npz: one step of the original propagate.m with its measurement-noise lines active,
composed from the reference's conlin.m, gp2.m, gSin.m and gp0.m (the checksummed copies under
tests/reference_tests/Matlab Code) EXECUTED with oracle/mrun.py, for a linear and an RBF policy (DESIGN.md section 22):

    ss = S + diag(sn2);  [Mp, Sp, Cp] = policy(m, ss);  [Mu, Su, C2] = gSin(Mp, Sp, maxU);  q = S Cp C2
    [Md, Sd, Cd] = gp0(dyn, [m; Mu], [S q; q' Su]);  Mnext = m + Md;  Snext = sym(S + Sd + Q + Q'),  Q = [S q] Cd

(difi = every dimension: all targets are differences; no angles).

    python tests/golden/make_obs_noise_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import mrun            # noqa: E402
from util import hyp_of, make_gp_problem   # noqa: E402


def step(policy, m, s, sn2, maxU, dyn):
    ss = s + np.diag(sn2)
    Mp, Sp, Cp = policy(m, ss)
    Mu, Su, C2 = mrun.run("gSin", np.asarray(Mp).reshape(-1, 1), np.asarray(Sp), float(maxU[0]), nout=3)
    q = s @ (np.asarray(Cp) @ np.asarray(C2))
    Mj = np.vstack([m.reshape(-1, 1), np.asarray(Mu).reshape(-1, 1)])
    Sj = np.block([[s, q], [q.T, np.asarray(Su)]])
    Md, Sd, Cd = mrun.run("gp0", dyn, Mj, Sj, nout=3)
    Q = Sj[:len(m)] @ np.asarray(Cd)
    Sn = s + np.asarray(Sd) + Q + Q.T
    return m.reshape(-1) + np.asarray(Md).reshape(-1), 0.5 * (Sn + Sn.T)


def main():
    out = {}
    Ds, U = 3, 2
    for case, seed in (("linear", 1), ("rbf", 2)):
        X, Y, ell, sf2, sn2d = make_gp_problem(40, Ds + U, Ds, seed=seed)
        Y = 0.1 * Y
        rng = np.random.RandomState(seed + 10)
        B = rng.randn(Ds, Ds)
        m, s = X[0, :Ds].copy(), 0.03 * B @ B.T + 0.02 * np.eye(Ds)
        sn2 = 0.01 + 0.05 * rng.rand(Ds)
        maxU = (0.7 + rng.rand()) * np.ones(U)            # gSin.m scales every action by one e
        dyn = dict(hyp=hyp_of(ell, sf2, sn2d), inputs=X, targets=Y)
        rec = dict(m=m, s=s, sn2=sn2, X=X, Y=Y, ell=ell, sf2=sf2, sn2_dyn=sn2d, maxU=maxU)
        if case == "linear":
            W, b = 0.5 * rng.randn(U, Ds), 0.3 * rng.randn(U)
            policy = lambda mm, sx: mrun.run("conlin", dict(p=dict(w=W, b=b.reshape(-1, 1))), mm.reshape(-1, 1), sx,
                                             nout=3)
            rec.update(W=W, b=b)
        else:
            Xc, Yc, lc = 0.5 * rng.randn(10, Ds) + 0.5, 0.1 * rng.randn(10, U), 1.0 + 0.1 * rng.randn(U, Ds)
            pol = dict(hyp=hyp_of(lc, np.ones(U), 1e-4 * np.ones(U)), inputs=Xc, targets=Yc)
            policy = lambda mm, sx: mrun.run("gp2", pol, mm.reshape(-1, 1), sx, nout=3)
            rec.update(Xc=Xc, Yc=Yc, lc=lc)
        rec["Mnext"], rec["Snext"] = step(policy, m, s, sn2, maxU, dyn)
        for k, v in rec.items():
            out["%s_%s" % (case, k)] = np.asarray(v, dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "obs_noise.npz"), **out)
    print("wrote obs_noise", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
