"""Torch statement of PILCO's gTrig stage in propagate.m, the moments of the angular feature map: written with the
second moments e+- = exp(-(s_aa + s_bb +- 2 s_ab)/2) as in the PILCO papers (the device writes them with expm1).
tests/action_reward_oracle.py puts it in front of the policy and the dynamics; autograd through it gives the
reference gradients."""
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
