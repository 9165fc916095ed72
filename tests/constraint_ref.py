"""An independent fp64 statement of the engine's soft-constraint problem, for test_cpu_constraint.py and test_gpu_constraint.py.

Written from the engine's documented definitions (the Computation chapter; SURVEY.md Appendix C), not from the oracle's or the
device's code, and organised differently on purpose: parameters per constraint, then rows, then one generic conjugate for every
constraint's force and cost.

- Contact parameters: the higher `priority` geom's condim, friction, solref and solimp; at equal priority condim = max,
  friction = element-wise max, the solmix weight, solref mixed by it when both time constants are positive (else element-wise
  min), solimp mixed by it.  A contact's five friction coefficients are (slide, slide, spin, roll, roll).
- Impedance: the two-piece power sigmoid of x = |pos - margin| / width between dmin and dmax.
- Reference acceleration aref = -B vel - K imp (pos - margin), K and B from solref (time constant and damping ratio, or direct
  stiffness and damping when negative); K = 0 on friction-loss rows and on the friction rows of a cone.
- Regularisation R = max(MINVAL, (1 - imp) / imp * diagApprox); on a cone R_1 = R_0 / impratio and R_k = R_1 mu_0^2 / mu_k^2.
- Force of a constraint block at x = J qacc - aref: f*(x) = argmax_{f in K} (-f.x - f.R.f / 2), with K = [-fl, fl] (friction
  loss), [0, inf) (limit, frictionless contact) or the elliptic cone {f_0 >= |(f_i / mu_i)|}.  The cone's maximiser is found as
  an R-weighted projection by a 1-D root find on its KKT multiplier; the engine's three cone zones are not used.
- Primal cost F(a) = (a - a_s).M.(a - a_s) / 2 + sum s(J a - aref), s(x) = -f*.x - f*.R.f* / 2, gradient
  g(a) = M a - qfrc_smooth - J^T f*(J a - aref).  F is 1-strongly convex in the M-norm, so for any a:
  |a - a*|_M <= |g(a)|_{M^-1} and F(a) - F* <= |g(a)|^2_{M^-1} / 2.  This certificate judges an answer without trusting a solver.
"""
import numpy as np

MINVAL = 1e-15
MINIMP, MAXIMP = 1e-4, 0.9999
FRICTION, LIMIT, FRICTIONLESS, ELLIPTIC = 1, 3, 5, 7  # efc_type codes


# ------------------------------------------------------------------------------------------------ parameters
def _clip(v, lo, hi):
    return min(max(float(v), lo), hi)


def power_sigmoid(x, mid, power):
    """0 at x = 0, 1 at x = 1, value `mid` at x = mid: x^p / mid^(p-1) below mid, mirrored above"""
    if x <= mid:
        return x ** power / mid ** (power - 1)
    return 1 - (1 - x) ** power / (1 - mid) ** (power - 1)


def impedance(solimp, pos, margin=0.0):
    """d(r) in [dmin, dmax] of a row at violation r = pos - margin"""
    dmin, dmax, mid = (_clip(solimp[k], MINIMP, MAXIMP) for k in (0, 1, 3))
    width, power = max(0.0, float(solimp[2])), max(1.0, float(solimp[4]))
    if dmin == dmax or width <= MINVAL:
        return (dmin + dmax) / 2
    x = abs(pos - margin) / width
    if x >= 1:
        return dmax
    return dmin + (dmax - dmin) * power_sigmoid(x, mid, power)


def stiffness_damping(solref, solimp, timestep):
    """(K, B) of aref = -B vel - K imp r"""
    dmax = _clip(solimp[1], MINIMP, MAXIMP)
    if solref[0] > 0:
        timeconst, dampratio = max(float(solref[0]), 2 * timestep), float(solref[1])
        return 1 / max(MINVAL, (dmax * timeconst * dampratio) ** 2), 2 / max(MINVAL, dmax * timeconst)
    return -solref[0] / max(MINVAL, dmax * dmax), -solref[1] / max(MINVAL, dmax)


def solmix_weight(s1, s2):
    if s1 < MINVAL and s2 < MINVAL:
        return 0.5
    if s1 < MINVAL:
        return 0.0
    if s2 < MINVAL:
        return 1.0
    return s1 / (s1 + s2)


def contact_params(model, g1, g2, env=None):
    """(condim, friction[5], solref[2], solimp[5]) of a contact between geoms g1 and g2; env: per-environment values (see Env)"""
    env = env or Env()
    fr = [np.asarray(env.geom_friction.get(g, model.geom_friction[g]), dtype=np.float64) for g in (g1, g2)]
    sr = [np.asarray(env.geom_solref.get(g, model.geom_solref[g]), dtype=np.float64) for g in (g1, g2)]
    si = [np.asarray(env.geom_solimp.get(g, model.geom_solimp[g]), dtype=np.float64) for g in (g1, g2)]
    p1, p2 = int(model.geom_priority[g1]), int(model.geom_priority[g2])
    if p1 != p2:
        w = 0 if p1 > p2 else 1
        condim, f3, solref, solimp = int(model.geom_condim[(g1, g2)[w]]), fr[w], sr[w], si[w]
    else:
        condim = max(int(model.geom_condim[g1]), int(model.geom_condim[g2]))
        f3 = np.maximum(fr[0], fr[1])
        mix = solmix_weight(float(model.geom_solmix[g1]), float(model.geom_solmix[g2]))
        solref = mix * sr[0] + (1 - mix) * sr[1] if sr[0][0] > 0 and sr[1][0] > 0 else np.minimum(sr[0], sr[1])
        solimp = mix * si[0] + (1 - mix) * si[1]
    return condim, np.array([f3[0], f3[0], f3[1], f3[2], f3[2]]), np.asarray(solref, dtype=np.float64), np.asarray(solimp, dtype=np.float64)


class Env:
    """per-environment model values (b2s_model_override) and the derived constants they imply; empty = the model's own"""

    def __init__(self, dof_frictionloss=None, geom_friction=None, geom_solref=None, geom_solimp=None, dof_invweight0=None,
                 body_invweight0=None, meaninertia=None):
        self.dof_frictionloss, self.dof_invweight0, self.body_invweight0, self.meaninertia = \
            dof_frictionloss, dof_invweight0, body_invweight0, meaninertia
        self.geom_friction, self.geom_solref, self.geom_solimp = geom_friction or {}, geom_solref or {}, geom_solimp or {}


# ------------------------------------------------------------------------------------------------ rows
class Block:
    """one constraint: rows [start, start + dim) of kind FRICTION / LIMIT / FRICTIONLESS / ELLIPTIC; `fl` the friction-loss bound,
    `mu` the dim - 1 friction coefficients of a cone"""

    def __init__(self, kind, start, dim, fl=0.0, mu=None, contact=-1):
        self.kind, self.start, self.dim, self.fl, self.mu, self.contact = kind, start, dim, fl, mu, contact

    @property
    def rows(self):
        return slice(self.start, self.start + self.dim)


class Rows:
    """the reference's constraint rows: type, J, aref, R, D, and the blocks"""

    def __init__(self, nv):
        self.nv = nv
        self.type, self.J, self.aref, self.R, self.blocks = [], [], [], [], []

    @property
    def nefc(self):
        return len(self.type)

    def add(self, kind, Jrows, aref, R, **kw):
        self.blocks.append(Block(kind, self.nefc, len(Jrows), **kw))
        self.type += [kind] * len(Jrows)
        self.J += list(Jrows)
        self.aref += list(aref)
        self.R += list(R)

    def arrays(self):
        J = np.array(self.J, dtype=np.float64).reshape(self.nefc, self.nv)
        R = np.array(self.R, dtype=np.float64)
        return np.array(self.type, dtype=int), J, np.array(self.aref, dtype=np.float64), R, 1 / R


def build_rows(model, o, env=None, max_rows=None):
    """rows of the oracle's current state (o.forward() done): friction loss per dof, limits per joint (lower side, then upper),
    contacts with all of their rows or none.  max_rows: capacity; a contact that does not fit is left out with the rest."""
    env = env or Env()
    nv, ts = model.nv, float(model.opt_timestep)
    qpos, qvel = np.array(o.qpos, dtype=np.float64), np.array(o.qvel, dtype=np.float64)
    dof_iw = np.asarray(env.dof_invweight0 if env.dof_invweight0 is not None else model.dof_invweight0, dtype=np.float64)
    body_iw = np.asarray(env.body_invweight0 if env.body_invweight0 is not None else model.body_invweight0,
                         dtype=np.float64).reshape(-1, 2)
    floss = np.asarray(env.dof_frictionloss if env.dof_frictionloss is not None else model.dof_frictionloss, dtype=np.float64)
    rows = Rows(nv)

    def unit(dof, sign):
        e = np.zeros(nv)
        e[dof] = sign
        return e

    def scalar_row(solref, solimp, r, margin, vel, diag, friction_row):
        imp = impedance(solimp, r, margin)
        K, B = stiffness_damping(solref, solimp, ts)
        if friction_row:
            K = 0.0
        return -B * vel - K * imp * (r - margin), max(MINVAL, (1 - imp) / imp * diag)

    for dof in range(nv):
        if floss[dof] > 0:
            aref, R = scalar_row(model.dof_solref[dof], model.dof_solimp[dof], 0.0, 0.0, qvel[dof], dof_iw[dof], True)
            rows.add(FRICTION, [unit(dof, 1.0)], [aref], [R], fl=float(floss[dof]))
    for j in range(model.njnt):
        if not model.jnt_limited[j] or int(model.jnt_type[j]) not in (2, 3):  # slide, hinge
            continue
        q, dof, margin = qpos[model.jnt_qposadr[j]], int(model.jnt_dofadr[j]), float(model.jnt_margin[j])
        lo, hi = model.jnt_range[j]
        for dist, sign in ((q - lo, 1.0), (hi - q, -1.0)):
            if dist < margin:
                aref, R = scalar_row(model.jnt_solref[j], model.jnt_solimp[j], dist, margin, sign * qvel[dof], dof_iw[dof], False)
                rows.add(LIMIT, [unit(dof, sign)], [aref], [R])
    impratio = float(model.opt_impratio)
    for ci, c in enumerate(o.contacts()):
        if c["dist"] >= 0:
            continue
        g1, g2 = c["geom1"], c["geom2"]
        condim, fr5, solref, solimp = contact_params(model, g1, g2, env)
        if max_rows is not None and rows.nefc + condim > max_rows:
            break
        b1, b2 = int(model.geom_bodyid[g1]), int(model.geom_bodyid[g2])
        p1, r1 = o.jac(c["pos"], b1)
        p2, r2 = o.jac(c["pos"], b2)
        frame = np.asarray(c["frame"], dtype=np.float64).reshape(3, 3)
        Jc = np.concatenate([frame @ (p2 - p1), frame @ (r2 - r1)])[:condim]
        vel = Jc @ qvel
        imp = impedance(solimp, c["dist"], 0.0)
        K, B = stiffness_damping(solref, solimp, ts)
        diag = [body_iw[b1, 0] + body_iw[b2, 0]] * 3 + [body_iw[b1, 1] + body_iw[b2, 1]] * 3
        R0 = max(MINVAL, (1 - imp) / imp * diag[0])
        aref = [-B * vel[0] - K * imp * c["dist"]] + [-B * v for v in vel[1:]]
        if condim == 1:
            rows.add(FRICTIONLESS, Jc, aref, [R0], contact=ci)
            continue
        R1 = R0 / max(MINVAL, impratio)
        mu = fr5[:condim - 1]
        rows.add(ELLIPTIC, Jc, aref, [R0] + [R1 * mu[0] ** 2 / m ** 2 for m in mu], mu=mu, contact=ci)
    return rows


# ------------------------------------------------------------------------------------------------ the conjugate
def cone_force(x, R, mu):
    """argmax over the cone {f_0 >= |(f_i / mu_i)|} of -f.x - f.R.f / 2 = the R-weighted projection of p = -x / R.  On the cone's
    surface, with multiplier lam = (t - p_0) R_0 >= 0 and t = f_0 > 0: f_i = p_i R_i mu_i^2 t / (R_i mu_i^2 t + lam), and t solves
    psi(t) = |(p_i R_i mu_i / (R_i mu_i^2 t + (t - p_0) R_0))| - 1 = 0, psi decreasing for t > max(0, p_0)."""
    from scipy.optimize import brentq

    x, R, mu = (np.asarray(v, dtype=np.float64) for v in (x, R, mu))
    p = -x / R
    p0, pt, R0, Rt = p[0], p[1:], R[0], R[1:]
    if p0 >= 0 and np.linalg.norm(pt / mu) <= p0:
        return p
    c = Rt * mu * mu

    def psi(t):
        return np.linalg.norm(pt * Rt * mu / (c * t + (t - p0) * R0)) - 1

    if p0 < 0 and psi(0.0) <= 0:
        return np.zeros_like(p)
    lo = p0 if p0 > 0 else (0.0 if p0 < 0 else 1e-300)  # p_0 = 0: psi is infinite at 0
    hi = max(2 * lo, abs(p0), float(np.linalg.norm(pt / mu)), 1e-300)
    while psi(hi) > 0:
        hi *= 2
    t = brentq(psi, lo, hi, xtol=1e-300, rtol=4 * np.finfo(float).eps, maxiter=1000)
    return np.concatenate([[t], pt * c * t / (c * t + (t - p0) * R0)])


def block_force(b, x, R):
    """f*(x) of one block (x, R: the block's rows)"""
    if b.kind == FRICTION:
        return np.clip(-x / R, -b.fl, b.fl)
    if b.kind in (LIMIT, FRICTIONLESS) or b.dim == 1:
        return np.maximum(0.0, -x / R)
    return cone_force(x, R, b.mu)


def forces(blocks, x, R):
    """f*(x) and the constraint cost sum s(x) over all blocks"""
    f = np.zeros_like(x)
    for b in blocks:
        f[b.rows] = block_force(b, x[b.rows], R[b.rows])
    return f, float(-(f @ x) - 0.5 * (f * R) @ f)


class Problem:
    """the primal problem min_a F(a) of one environment"""

    def __init__(self, M, qfrc_smooth, J, aref, R, blocks, meaninertia):
        self.M, self.qs = np.asarray(M, dtype=np.float64), np.asarray(qfrc_smooth, dtype=np.float64)
        self.J, self.aref, self.R = (np.asarray(v, dtype=np.float64) for v in (J, aref, R))
        self.blocks = blocks
        self.nv = len(self.qs)
        self.a_s = np.linalg.solve(self.M, self.qs)
        self.scale = 1.0 / (float(meaninertia) * max(self.nv, 1))

    def force(self, a):
        return forces(self.blocks, self.J @ a - self.aref, self.R)[0]

    def cost(self, a):
        d = a - self.a_s
        return 0.5 * d @ self.M @ d + forces(self.blocks, self.J @ a - self.aref, self.R)[1]

    def grad(self, a):
        return self.M @ a - self.qs - self.J.T @ self.force(a)

    def certificate(self, a):
        """(|a - a*|_M bound, F(a) - F* bound in the solver's scaled units 1 / (meaninertia nv))"""
        g = self.grad(a)
        gn2 = float(g @ np.linalg.solve(self.M, g))
        return np.sqrt(max(gn2, 0.0)), self.scale * 0.5 * gn2

    def _force_jacobian(self, x):
        """-df*/dx block by block, central differences (the Newton polish only needs a fair model of the curvature)"""
        G = np.zeros((len(x), len(x)))
        for b in self.blocks:
            s = b.rows
            xs, Rs = x[s], self.R[s]
            for k in range(b.dim):
                h = 1e-7 * max(1.0, abs(xs[k]))
                e = np.zeros(b.dim)
                e[k] = h
                G[s, s.start + k] = -(block_force(b, xs + e, Rs) - block_force(b, xs - e, Rs)) / (2 * h)
        return G

    def solve(self, a0=None, target=1e-12):
        """a* by L-BFGS, then Newton steps on a finite-difference generalised Hessian with an exact line search.  Raises unless
        the answer's own certificate is below `target` (scaled cost gap)."""
        from scipy.optimize import minimize, minimize_scalar

        a = self.a_s.copy() if a0 is None else np.asarray(a0, dtype=np.float64).copy()
        if self.J.shape[0] == 0:
            return a
        r = minimize(lambda v: (self.cost(v), self.grad(v)), a, jac=True, method="L-BFGS-B",
                     options=dict(maxiter=5000, maxcor=30, ftol=0.0, gtol=0.0))
        a = r.x
        best = self.certificate(a)[1]
        for _ in range(60):
            if best < 1e-30:
                break
            x = self.J @ a - self.aref
            H = self.M + self.J.T @ self._force_jacobian(x) @ self.J
            d = np.linalg.solve(H + 1e-14 * np.trace(self.M) / self.nv * np.eye(self.nv), -self.grad(a))
            ls = minimize_scalar(lambda t: self.cost(a + t * d), bounds=(0.0, 2.0), method="bounded", options=dict(xatol=1e-14))
            cand = a + ls.x * d
            c_cand = self.certificate(cand)[1]
            full = a + d
            c_full = self.certificate(full)[1]
            if c_full < c_cand:
                cand, c_cand = full, c_full
            if c_cand >= best:
                break
            a, best = cand, c_cand
        if not best < target:
            raise AssertionError("reference minimiser: certificate %.3g above %.3g" % (best, target))
        return a


def problem_from_rows(rows, M, qfrc_smooth, meaninertia):
    _, J, aref, R, _ = rows.arrays()
    return Problem(M, qfrc_smooth, J, aref, R, rows.blocks, meaninertia)


def feasibility_violation(blocks, f):
    """largest violation of K by the forces f (0 when feasible), relative to the block's force scale"""
    worst = 0.0
    for b in blocks:
        fb = f[b.rows]
        sc = max(1.0, np.abs(fb).max())
        if b.kind == FRICTION:
            worst = max(worst, (np.abs(fb).max() - b.fl) / sc)
        elif b.kind in (LIMIT, FRICTIONLESS) or b.dim == 1:
            worst = max(worst, -fb.min() / sc)
        else:
            worst = max(worst, (np.linalg.norm(fb[1:] / b.mu) - fb[0]) / sc)
    return max(worst, 0.0)
