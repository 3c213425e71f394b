"""Torch statement of the moment-matching rollout with angular state dimensions (PILCO's gTrig stage in propagate.m):
the feature map's moments written with the second moments e+- = exp(-(s_aa + s_bb +- 2 s_ab)/2) as in the PILCO
papers (the device writes them with expm1), and the cascade of oracle/torch_port.py with that stage in front of the
policy and the dynamics.  Autograd through it gives the reference gradients."""
import torch

F64 = torch.float64


def trig_moments(m, s, angle_dims):
    """m [Ds], s [Ds,Ds] (torch) -> M [Dh], S [Dh,Dh], C = inv(s) cov(x, phi) [Ds,Dh]"""
    Ds = m.shape[0]
    dims = [int(a) for a in angle_dims]
    keep = [j for j in range(Ds) if j not in dims]
    A = len(dims)
    Dh = Ds + A
    ea = [torch.exp(-0.5 * s[a, a]) for a in dims]
    Es = [ea[i] * torch.sin(m[a]) for i, a in enumerate(dims)]
    Ec = [ea[i] * torch.cos(m[a]) for i, a in enumerate(dims)]
    M = torch.cat([m[keep]] + [torch.stack([Es[i], Ec[i]]) for i in range(A)])
    # columns of phi: (state dim, kind) with kind 0 pass, 1 sin, 2 cos
    cols = [(j, 0) for j in keep] + [(a, k) for a in dims for k in (1, 2)]
    idx = {a: i for i, a in enumerate(dims)}
    rows = []
    for (i, ki) in cols:
        row = []
        for (j, kj) in cols:
            if ki == 0 and kj == 0:
                v = s[i, j]
            elif ki == 0 or kj == 0:
                a, kind = (j, kj) if ki == 0 else (i, ki)
                v = s[i, j] * (Ec[idx[a]] if kind == 1 else -Es[idx[a]])
            else:
                em = torch.exp(-0.5 * (s[i, i] + s[j, j] - 2 * s[i, j]))
                ep = torch.exp(-0.5 * (s[i, i] + s[j, j] + 2 * s[i, j]))
                mi, mj = m[i], m[j]
                if ki == 1 and kj == 1:
                    e2 = 0.5 * (em * torch.cos(mi - mj) - ep * torch.cos(mi + mj))
                elif ki == 2 and kj == 2:
                    e2 = 0.5 * (em * torch.cos(mi - mj) + ep * torch.cos(mi + mj))
                elif ki == 1:
                    e2 = 0.5 * (ep * torch.sin(mi + mj) + em * torch.sin(mi - mj))
                else:
                    e2 = 0.5 * (ep * torch.sin(mj + mi) + em * torch.sin(mj - mi))
                mu_i = Es[idx[i]] if ki == 1 else Ec[idx[i]]
                mu_j = Es[idx[j]] if kj == 1 else Ec[idx[j]]
                v = e2 - mu_i * mu_j
            row.append(v)
        rows.append(torch.stack(row))
    S = torch.stack(rows)
    C = torch.zeros((Ds, Dh), dtype=F64)
    Ccols = []
    for k, (d, kind) in enumerate(cols):
        col = torch.zeros(Ds, dtype=F64)
        onehot = torch.zeros(Ds, dtype=F64)
        onehot[d] = 1.0
        if kind == 0:
            col = onehot
        elif kind == 1:
            col = onehot * Ec[idx[d]]
        else:
            col = onehot * (-Es[idx[d]])
        Ccols.append(col)
    C = torch.stack(Ccols, dim=1)
    return M, S, C


def propagate(m_x, s_x, angle_dims, action_fn, dynamics_fn):
    """one step: m_x [1,Ds], s_x [Ds,Ds] -> (next m [1,Ds], next s, joint m [1,D], joint s [D,D])"""
    mh, Sh, Ch = trig_moments(m_x[0], s_x, angle_dims)
    mh = mh[None]
    m_u, s_u, c_xu = action_fn(mh, Sh)
    m = torch.cat([mh, m_u], dim=1)
    s1 = torch.cat([Sh, Sh @ c_xu], dim=1)
    s2 = torch.cat([(Sh @ c_xu).T, s_u], dim=1)
    s = torch.cat([s1, s2], dim=0)
    M_dx, S_dx, C_dx = dynamics_fn(m, s)
    Q = s_x @ Ch
    cxx = torch.cat([Q, Q @ c_xu], dim=1)             # cov(x, [phi, u])
    K = cxx @ C_dx
    return M_dx + m_x, S_dx + s_x + K + K.T, m, s


def predict(m_x, s_x, n, angle_dims, action_fn, dynamics_fn, reward_fn, joint_reward_fn=None):
    """H-step cascade: returns (trajectory means [n+1,Ds], covariances [n+1,Ds,Ds], total reward)"""
    total = torch.zeros((), dtype=F64)
    ms, Ss = [m_x[0]], [s_x]
    for _ in range(n):
        r = reward_fn(m_x, s_x).reshape(())
        m_x, s_x, mj, sj = propagate(m_x, s_x, angle_dims, action_fn, dynamics_fn)
        if joint_reward_fn is not None:
            r = r + joint_reward_fn(mj, sj).reshape(())
        total = total + r
        ms.append(m_x[0]); Ss.append(s_x)
    return torch.stack(ms), torch.stack(Ss), total
