"""Extended-precision reference of the basis and deterministic-signal kernels -- ``ptar_fourier_basis``,
``ptar_cholesky_lower``, ``ptar_cgw_delay``, ``ptar_cw_catalog`` (prefactors, sources x TOAs, slice reduction),
``ptar_burst_delay`` and ``ptar_memory_delay`` -- with a first-order componentwise error bound per output that holds
for any evaluation order and any FMA contraction; numpy only, no torch.

The reference evaluates the operation each kernel performs on the fp64 operands the kernel receives (the Fourier rows
rebuilt from ``plan()``, the ORF as uploaded, ``PulsarBatch.cgw_inputs``, the catalog and the device's own ``pre``),
so only kernel arithmetic is under test; the physics is the oracle tests' business.

Error-carrying evaluator.  ``E`` carries (value in np.longdouble, absolute bound in fp64) through the kernel's own
sequence of operations, u = 2^-53:
  add / sub   e = e_x + e_y + u |v|
  mul         e = |y| e_x + |x| e_y + u |v|           (a power-of-two or zero fp64 constant: exact, e = |c| e_x)
  div         e = (e_x + |v| e_y) / |y| + u |v|
  f(x)        e = |f'(x)| e_x + k_f 2u |v|           (sin, cos: + e_x^2 / 2, so the bound stays valid where f' ~ 0)
with k_f the maximum ulp error of CUDA's double functions: sin, cos, sincos 2; pow 2; cbrt 1; sqrt 0 (IEEE).
Assumptions:
* the k_f are CUDA's documented maximum errors (CUDA C++ Programming Guide, "Mathematical Functions"); they were not
  measured here;
* double ``/`` and ``sqrt`` are IEEE (correctly rounded) under the project's ``-prec-div=false -prec-sqrt=false
  -ftz=true``: those flags only touch fp32 (see ``__graft_entry__.py``);
* the separate-rounding rule for ``a * b + c`` also bounds its FMA-contracted form (one rounding fewer);
* the longdouble value (64-bit mantissa) of each operation is within 2^-11 of its bound term, so the reference itself
  is exact to ~5e-4 of the bound (tests/test_deterministic_edges_cpu.py checks it against mpmath at 40 digits).
The kernels' fp64 constants are used, not the exact ones: ``pow(x, fl(-5/3))``, fl(pi), fl(2 pi) = 6.283185307179586,
and the SOLAR2S, MPC2S and KPC2S literals.  A pow with the exact exponent moves the worst output of the CW sweep's
sources by 1.27 times its bound (the margin is small because pow's documented 2 ulp dominate the phase bound), so a
reference with the exact constants would fail a correct kernel.

Bounds per family:
* Fourier basis: arg = fl(fl(2 pi) t) f (+ phase), then sin / cos; every Ftile entry is rebuilt from
  plan()["tiles"], ep_tref, t0_table, freqs and conv, and rows past a tile's epoch count must be exactly 0.
* Cholesky (Higham, Accuracy and Stability of Numerical Algorithms, Theorem 10.3): |A - L L^T| <= gamma_{n+1}
  |L| |L^T|, the product in pair arithmetic; strict upper triangle exactly 0, diagonal > 0, info = 0.
* CW: one formula (``cw_res``) mirrors cgw_kernel / cw_catalog_kernel line by line for all three modes and both
  psr_term values; catalog prefactors (``prefactors``) mirror cw_prefactor_kernel.  The catalog sum over sources
  and slices: out = sum_s r_s with |d| <= sum_s e_s + gamma_{n_src (+1 with accumulate)} (sum_s |r_s| + |out_0|);
  a source whose value is NaN contributes exactly 0.
* Burst and memory: bit-exact against numpy fp64 (the kernels round every product with __dmul_rn / __dsub_rn)."""
from __future__ import annotations

import math

import numpy as np

from tests.reduction_reference import U, Report, check, gamma, xmatmul  # noqa: F401

LD = np.longdouble
PI = 3.141592653589793                 # fl(pi), the kernels' literal
TWO_PI = 6.283185307179586             # fl(2 pi) = 2 fl(pi)
SOLAR2S = 4.925838061995516e-06        # cw_prefactor_kernel's literals (constants.py)
MPC2S = 102927125054338.98
KPC2S = 102927125054.33899
K_SIN, K_POW, K_CBRT = 2, 2, 1         # CUDA double max ulp errors: sin / cos / sincos, pow, cbrt


# ------------------------------------------------------------------ error-carrying evaluator
def _exact_const(c):
    """A Python / numpy fp64 scalar whose products are exact: 0 or a power of two."""
    return isinstance(c, (float, int, np.floating)) and (c == 0 or abs(math.frexp(float(c))[0]) == 0.5)


def _r(v):
    return U * np.abs(v).astype(np.float64)


class E:
    """(value in longdouble, absolute error bound in fp64), elementwise over broadcastable arrays."""
    __array_priority__ = 100

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=LD)
        self.e = np.zeros(self.v.shape) if e is None else np.asarray(e, dtype=np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(np.asarray(x, dtype=np.float64))

    def __add__(self, o):
        o = E.of(o)
        v = self.v + o.v
        return E(v, self.e + o.e + _r(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = E.of(o)
        v = self.v - o.v
        return E(v, self.e + o.e + _r(v))

    def __rsub__(self, o):
        return E.of(o) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        if _exact_const(o):
            return E(self.v * LD(float(o)), self.e * abs(float(o)))
        o = E.of(o)
        v = self.v * o.v
        return E(v, np.abs(o.v).astype(np.float64) * self.e + np.abs(self.v).astype(np.float64) * o.e + _r(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        if _exact_const(o) and o != 0:
            return E(self.v / LD(float(o)), self.e / abs(float(o)))
        o = E.of(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            e = (self.e + np.abs(v).astype(np.float64) * o.e) / np.abs(o.v).astype(np.float64) + _r(v)
        return E(v, e)

    def __rtruediv__(self, o):
        return E.of(o) / self

    def out(self):
        """The check dict of reduction_reference.check: value as a pair hi + lo, bound, |value|."""
        hi = self.v.astype(np.float64)
        with np.errstate(invalid="ignore"):
            lo = np.where(np.isfinite(hi), (self.v - hi.astype(LD)).astype(np.float64), 0.0)
        return dict(hi=hi, lo=lo, bound=self.e, terms=np.abs(hi))


class EK:
    """Evaluator kit: the kernels' math functions on ``E``."""
    c = staticmethod(E.of)

    @staticmethod
    def sin(x):
        v = np.sin(x.v)
        return E(v, np.abs(np.cos(x.v)).astype(np.float64) * x.e + 0.5 * x.e * x.e + K_SIN * 2 * _r(v))

    @staticmethod
    def cos(x):
        v = np.cos(x.v)
        return E(v, np.abs(np.sin(x.v)).astype(np.float64) * x.e + 0.5 * x.e * x.e + K_SIN * 2 * _r(v))

    @staticmethod
    def pow(x, c):
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            v = np.power(x.v, LD(c))
            d = np.abs(LD(c) * v / x.v).astype(np.float64)
        return E(v, d * x.e + K_POW * 2 * _r(v))

    @staticmethod
    def cbrt(x):
        v = np.cbrt(x.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            d = np.abs(v / (3 * x.v)).astype(np.float64)
        return E(v, d * x.e + K_CBRT * 2 * _r(v))

    @staticmethod
    def sqrt(x):
        v = np.sqrt(x.v)
        return E(v, x.e / (2 * v.astype(np.float64)) + _r(v))


class NK:
    """numpy fp64 kit: the same formulas evaluated the way a kernel would (mutants are built on it)."""
    c = staticmethod(np.float64)
    sin, cos, cbrt, sqrt = np.sin, np.cos, np.cbrt, np.sqrt

    @staticmethod
    def pow(x, c):
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.power(x, c)

    @staticmethod
    def pow_exact53(x):
        """x^(-5/3) with the exact exponent, rounded once (the mutant of fl(-5/3))."""
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.power(np.asarray(x, dtype=LD), LD(-5) / LD(3)).astype(np.float64)


class MK:
    """mpmath kit (scalar points), for checking the longdouble reference itself."""
    import mpmath as _mp
    mp = _mp
    c = staticmethod(lambda x: MK.mp.mpf(float(x)))
    sin = staticmethod(lambda x: MK.mp.sin(x))
    cos = staticmethod(lambda x: MK.mp.cos(x))
    cbrt = staticmethod(lambda x: MK.mp.cbrt(x))
    sqrt = staticmethod(lambda x: MK.mp.sqrt(x))
    pow = staticmethod(lambda x, c: MK.mp.power(x, MK.mp.mpf(float(c))))


# ------------------------------------------------------------------ Fourier basis
def fourier_arg(K, t, f, phase=None):
    """fourier_basis_kernel's argument: fl(fl(2 pi) t) f (+ phase)."""
    a = (K.c(TWO_PI) * t) * f
    return a if phase is None else a + phase


def fourier_rows(pl, t0_table, conv):
    """Per Ftile row (tile epoch): (tile, epoch in tile, pulsar, t) from plan()["tiles"], ep_tref and t0_table."""
    ti, ee, pp, tt = [], [], [], []
    for k, (_, _, _, ep0, nep, psr, _, _) in enumerate(np.asarray(pl["tiles"]).tolist()):
        tr = pl["ep_tref"][ep0:ep0 + nep]
        ti.append(np.full(nep, k)); ee.append(np.arange(nep)); pp.append(np.full(nep, psr))
        tt.append(tr - t0_table[psr] if conv else tr)       # the host's fp64 subtraction: an exact kernel operand
    return tuple(np.concatenate(a) for a in (ti, ee, pp, tt))


def ftile(pl, t0_table, conv, K=EK, mut=()):
    """Ftile [n_tiles * J * 64] (check dict for ``K = EK``, fp64 for ``NK``).  ``mut`` (NK only): "swap" sin / cos,
    "nbr_freq" the first tile of pulsar 1 takes pulsar 2's frequencies, "row_shift" a 17- or 33-epoch tile's rows
    take the next epoch's time."""
    J, EPN = pl["J"], 64
    nk = J // 2
    ti, ee, pp, tt = fourier_rows(pl, t0_table, conv)
    freqs = np.asarray(pl["freqs"], dtype=np.float64)
    fr = freqs[pp]
    if "nbr_freq" in mut:
        first = int(np.flatnonzero(pp == 1)[0])
        rows = (ti == ti[first])
        fr[rows] = freqs[2]
    if "row_shift" in mut:
        nep = np.asarray(pl["tiles"])[:, 4]
        k = int(np.flatnonzero((nep == 17) | (nep == 33))[0])
        rows = np.flatnonzero(ti == k)
        tt = tt.copy()
        tt[rows[:-1]] = tt[rows[1:]]
    a = fourier_arg(K, K.c(tt)[:, None] if K is not EK else E(tt[:, None]), K.c(fr) if K is not EK else E(fr))
    s, c = K.sin(a), K.cos(a)
    if "swap" in mut:
        s, c = c, s
    first_col, second_col = (c, s) if conv else (s, c)
    idx = (ti * J * EPN + ee)[:, None] + (np.arange(nk) * 2 * EPN)[None, :]
    n = len(pl["tiles"]) * J * EPN
    if K is EK:
        out = dict(hi=np.zeros(n), lo=np.zeros(n), bound=np.zeros(n), terms=np.zeros(n))
        for col, off in ((first_col, 0), (second_col, EPN)):
            o = col.out()
            for key in out:
                out[key][idx + off] = o[key]
        return out
    F = np.zeros(n)
    F[idx] = first_col
    F[idx + EPN] = second_col
    return F


def design_matrix(t, f, phase, conv, K=EK):
    """create_fourier_design_matrix_red's kernel call: F [N, 2 nmodes] (col_stride 1)."""
    tp = t - t[0] if conv else t
    a = fourier_arg(K, E(tp[:, None]) if K is EK else tp[:, None], E(f) if K is EK else f,
                    None if phase is None else (E(phase) if K is EK else phase))
    s, c = K.sin(a), K.cos(a)
    first, second = (c, s) if conv else (s, c)
    if K is not EK:
        out = np.empty((len(t), 2 * len(f)))
        out[:, 0::2], out[:, 1::2] = first, second
        return out
    o1, o2 = first.out(), second.out()
    res = {}
    for key in o1:
        res[key] = np.empty((len(t), 2 * len(f)))
        res[key][:, 0::2], res[key][:, 1::2] = o1[key], o2[key]
    return res


# ------------------------------------------------------------------ Cholesky
def cholesky_ref(A, L):
    """Check dict of Higham's Theorem 10.3 over the lower triangle: compare ``A`` (as ``dev``) with the pair L L^T,
    bound gamma_{n+1} |L| |L^T|; the upper triangle is masked out (0 = 0)."""
    n = A.shape[-1]
    h, l = xmatmul(L, L.T)
    t = np.abs(L) @ np.abs(L.T)
    low = np.tril(np.ones((n, n), dtype=bool))
    return dict(hi=np.where(low, h, A), lo=np.where(low, l, 0.0), bound=np.where(low, gamma(n + 1) * t, 0.0), terms=t)


def cholesky_np(A, mut=()):
    """Left-looking Cholesky in numpy fp64 (the mutants' base): "nodiv_last" the last column with sub-diagonal
    entries is not divided by l_jj, "no_sqrt" the last diagonal takes d in place of sqrt(d)."""
    n = A.shape[0]
    L = np.tril(A).astype(np.float64)
    for j in range(n):
        d = L[j, j] - L[j, :j] @ L[j, :j]
        ljj = d if ("no_sqrt" in mut and j == n - 1) else np.sqrt(d)
        for i in range(j + 1, n):
            v = L[i, j] - L[i, :j] @ L[j, :j]
            L[i, j] = v if ("nodiv_last" in mut and j == n - 2) else v / ljj
        L[j, j] = ljj
    return L


def spd(n, kappa, rng):
    """A random symmetric positive definite matrix of condition number ~``kappa`` (log-spaced spectrum)."""
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.logspace(0, -np.log10(kappa), n) if n > 1 else np.ones(1)
    A = (Q * lam) @ Q.T
    return 0.5 * (A + A.T)


def not_pd_at(n, k, rng):
    """A symmetric matrix whose leading minors 1 .. k-1 are positive definite and whose minor k is the first that is
    not: A = L0 L0^T with A[k-1][k-1] lowered by L0[k-1][k-1]^2 + 1 (Schur complement ~ -1)."""
    L0 = np.tril(rng.uniform(-0.5, 0.5, (n, n)) / np.sqrt(n), -1) + np.eye(n)
    A = L0 @ L0.T
    A = 0.5 * (A + A.T)
    A[k - 1, k - 1] -= L0[k - 1, k - 1] ** 2 + 1.0
    return A


def ng15_radec(kind="full", seed=20250922, npsr=67):
    """(RA, DEC) [rad] of synthetic.make_ng15_like(kind): its random stream replayed without building the TOAs."""
    from pta_replicator_b200 import noise_dict as nd
    names = nd.pulsar_names(nd.load_noise_dict())[:npsr]
    rng = np.random.default_rng(seed)
    out = np.zeros((len(names), 2))
    for i, _ in enumerate(names):
        nep = int(rng.integers(100, 501))
        nsub = int(rng.integers(10, 61)) if kind == "full" else 1
        rng.uniform(53000.0, 58800.0, nep)
        rng.uniform(0.0, 0.5, (nep, nsub))
        rng.uniform(0.1, 3.0, nep * nsub)
        raj = float(rng.uniform(0.0, 24.0))
        decj = float(np.degrees(np.arcsin(rng.uniform(-1.0, 1.0))))
        out[i] = raj * np.pi / 12.0, decj * np.pi / 180.0
    return out


def orf_matrix(radec, clm=(math.sqrt(4 * math.pi),), lmax=0):
    """The ORF ``PulsarBatch.set_gwb`` builds (2 sum_k clm[k] basis[k])."""
    from pta_replicator_b200 import orf as orf_mod
    locs = np.stack([radec[:, 0], np.pi / 2.0 - radec[:, 1]], axis=1)
    basis = orf_mod.correlated_basis(locs, lmax)
    return 2.0 * sum(clm[k] * basis[k] for k in range(len(basis)))


def config4_orf():
    """The lmax = 6 anisotropic ORF of test_gpu_parity.test_config4 (ng15-epoch sky, clm redrawn until PD)."""
    radec = ng15_radec("epoch")
    rng = np.random.default_rng(6)
    for _ in range(20):
        clm = np.r_[np.sqrt(4 * np.pi), 0.05 * rng.standard_normal(48)]
        orf = orf_matrix(radec, list(clm), 6)
        if np.all(np.linalg.eigvalsh(orf) > 1e-6):
            break
    return orf


# ------------------------------------------------------------------ continuous waves
def cw_res(K, toa, q, mode, psr_term, mut=()):
    """cgw_kernel / cw_catalog_kernel for one source: ``q`` = (w0, fac1, fac2, fac3, phase0, w053, incfac1, incfac2,
    cos2psi, sin2psi, fplus, fcross, cosMu, pd [s]).  Mutants (``mut``): "psr_sign" the pulsar term enters with the
    wrong sign, "tp_plus" 1 + cosMu in tp, "cbrt_omega" cbrt(omega) in place of cbrt(omega_p), "exact53" pow with
    the exact -5/3 (NK only)."""
    w0, fac1, fac2, fac3, phase0, w053, inc1, inc2, c2p, s2p, fplus, fcross, cosMu, pd = q
    p53 = K.pow_exact53 if "exact53" in mut else (lambda x: K.pow(x, -5.0 / 3))
    tp = toa - pd * ((1 + cosMu) if "tp_plus" in mut else (1 - cosMu))
    if mode == 0:
        omega = w0 * K.pow(1 - fac1 * toa, -3.0 / 8)
        omega_p = w0 * K.pow(1 - fac1 * tp, -3.0 / 8)
        phase = phase0 + fac2 * (w053 - p53(omega))
        phase_p = phase0 + fac2 * (w053 - p53(omega_p))
    elif mode == 1:
        omega = w0
        omega_p = w0 * K.pow(1 + fac1 * pd * (1 - cosMu), -3.0 / 8)
        phase = phase0 + omega * toa
        phase_p = phase0 + fac2 * (w053 - p53(omega_p)) + omega_p * toa
    else:
        omega = omega_p = w0
        phase = phase0 + omega * toa
        phase_p = phase0 + omega * tp
    At, Bt = K.sin(2 * phase) * inc1, K.cos(2 * phase) * inc2
    Atp, Btp = K.sin(2 * phase_p) * inc1, K.cos(2 * phase_p) * inc2
    alpha = fac3 / K.cbrt(omega)
    alpha_p = fac3 / K.cbrt(omega if "cbrt_omega" in mut else omega_p)
    rplus, rcross = alpha * (At * c2p + Bt * s2p), alpha * (-At * s2p + Bt * c2p)
    rplus_p, rcross_p = alpha_p * (Atp * c2p + Btp * s2p), alpha_p * (-Atp * s2p + Btp * c2p)
    if not psr_term:
        return -fplus * rplus - fcross * rcross
    if "psr_sign" in mut:
        return fplus * (-rplus_p - rplus) + fcross * (-rcross_p - rcross)
    return fplus * (rplus_p - rplus) + fcross * (rcross_p - rcross)


def cgw_ref(a, K=EK, mut=(), sel=slice(None)):
    """``det`` slots of ptar_cgw_delay from ``PulsarBatch.cgw_inputs`` (``a``), slots ``sel``."""
    par = a["par"][a["pid"][sel]]
    q = [K.c(a["src"][k]) for k in range(10)] + [K.c(par[:, k]) for k in range(4)]
    return cw_res(K, K.c(a["t"][sel]), q, a["mode"], a["psr_term"], mut)


def prefactors(K, cat, phat, pdist_kpc, pphase, use_pphase, mut=()):
    """cw_prefactor_kernel: pre[s][0..13] from ``cat`` [8, n_src] (gwtheta, gwphi, mc, dist, fgw, phase0, psi, inc)
    and the pulsar direction ``phat``.  Mutants: "phase0_full" phase0 not halved, "swap_fpc" fplus / fcross swapped."""
    gwtheta, gwphi, mcin, distin, fgw, ph0in, psi, inc = (K.c(cat[k]) for k in range(8))
    px, py, pz = (K.c(x) for x in phat)
    mc = mcin * SOLAR2S
    dist = distin * MPC2S
    phase0 = ph0in if "phase0_full" in mut else ph0in / 2
    w0 = PI * fgw
    cgt, cgp, sgt, sgp = K.cos(gwtheta), K.cos(gwphi), K.sin(gwtheta), K.sin(gwphi)
    mx, my = sgp, -cgp
    nx, ny, nz = -cgt * cgp, -cgt * sgp, sgt
    ox, oy, oz = -sgt * cgp, -sgt * sgp, -cgt
    mc53 = K.pow(mc, 5.0 / 3)
    mdp = mx * px + my * py + 0.0 * pz
    ndp = nx * px + ny * py + nz * pz
    odp = ox * px + oy * py + oz * pz
    cosMu = -odp
    pd = (K.c(pphase) / (TWO_PI * fgw * (1 - cosMu)) / KPC2S) if use_pphase else K.c(pdist_kpc)
    pd = pd * KPC2S
    fplus = 0.5 * (mdp * mdp - ndp * ndp) / (1 + odp)
    fcross = (mdp * ndp) / (1 + odp)
    if "swap_fpc" in mut:
        fplus, fcross = fcross, fplus
    return [w0, 256.0 / 5 * mc53 * K.pow(w0, 8.0 / 3), 1.0 / 32 / mc53, mc53 / dist, phase0, K.pow(w0, -5.0 / 3),
            0.5 * (3 + K.cos(2 * inc)), 2 * K.cos(inc), K.cos(2 * psi), K.sin(2 * psi), fplus, fcross, cosMu, pd]


def prefactors_np(cat, phat, pdist_kpc, pphase, use_pphase, mut=()):
    """cw_prefactor_kernel in numpy fp64: pre [n_src, 14]."""
    n = np.asarray(cat).shape[1]
    return np.stack([np.broadcast_to(x, (n,)) for x in prefactors(NK, cat, phat, pdist_kpc, pphase, use_pphase, mut)], axis=1)


def pre_ref(cat, phat, pdist_kpc, pphase, use_pphase):
    """Check dict over pre [n_src, 14]."""
    outs = [x.out() for x in prefactors(EK, cat, phat, pdist_kpc, pphase, use_pphase)]
    n = np.asarray(cat).shape[1]
    return {k: np.stack([np.broadcast_to(o[k], (n,)) for o in outs], axis=1) for k in outs[0]}


def catalog_sum_ref(pre, t, mode, psr_term, out0=None, chunk=2048):
    """out over the TOAs ``t`` = sum_s r_s (the device's ``pre`` [n_src, >= 14] as input; NaN sources contribute 0),
    bound sum_s e_s + gamma_{n_src (+1)} (sum_s |r_s| + |out0|).  Returns the check dict and the per-source
    values [n_src, n_t] (fp64, NaN kept) for the summation mutants."""
    n_src = pre.shape[0]
    v, e, a = np.zeros(len(t), dtype=LD), np.zeros(len(t)), np.zeros(len(t))
    rs = np.empty((n_src, len(t)))
    for s0 in range(0, n_src, chunk):
        q = [E(pre[s0:s0 + chunk, k][:, None]) for k in range(14)]
        r = cw_res(EK, E(t[None, :]), q, mode, psr_term)
        bad = np.isnan(r.v)
        rv = np.where(bad, LD(0), r.v)
        v += rv.sum(axis=0)
        e += np.where(bad, 0.0, r.e).sum(axis=0)
        a += np.abs(rv).astype(np.float64).sum(axis=0)
        rs[s0:s0 + chunk] = r.v.astype(np.float64)
    g = gamma(n_src)
    if out0 is not None:
        v += np.asarray(out0, dtype=LD)
        a += np.abs(out0)
        g = gamma(n_src + 1)
    res = E(v, e + g * a).out()
    res["terms"] = a
    return res, rs


def catalog_sum_np(rs, n_slices, out0=None, mut=()):
    """The device's summation order on fp64 source values ``rs`` [n_src, n_t]: 32-source stages within a slice, slices
    summed in order.  Mutants: "drop32" the 32nd source of each full stage is skipped, "twice" the second non-empty
    slice's partial is added twice, "nan" NaN sources are summed as NaN."""
    n_src = rs.shape[0]
    per = -(-n_src // n_slices)
    out = np.zeros(rs.shape[1])
    done = 0
    for k in range(n_slices):
        acc = np.zeros(rs.shape[1])
        for s in range(k * per, min(n_src, (k + 1) * per)):
            if "drop32" in mut and (s - k * per) % 32 == 31:
                continue
            r = rs[s]
            acc = acc + (r if "nan" in mut else np.where(np.isnan(r), 0.0, r))
        out = out + acc
        if k * per < n_src:
            done += 1
            if "twice" in mut and done == 2:
                out = out + acc
    return out if out0 is None else out0 + out


def check_nan(dev, ref, what="", report=None, family=None):
    """``check`` where an output that is NaN, or the same infinity, in both the device result and the reference counts
    as agreement."""
    dev = np.asarray(dev, dtype=np.float64)
    both = (np.isnan(dev) & np.isnan(ref["hi"])) | (np.isinf(dev) & (dev == ref["hi"]))
    r = {k: np.where(both, 0.0, v) for k, v in ref.items()}
    return check(np.where(both, 0.0, dev), r, what, report, family)


# ------------------------------------------------------------------ Fourier sweep batches
FOURIER_K = (1, 2, 10, 30, 129)
# (TOAs, span [days]) of the per-pulsar-Tspan batch: 1 / T from ~1 / (16 yr) to ~1 / (3 s), so that with conv = 0
# (t ~ 4.6e9 s) the arguments spread from ~1e2 to above 1e10 rad
OWN_SPANS = ((40, 5800.0), (30, 365.0), (20, 30.0), (12, 1.0), (6, 1.0 / 24), (3, 30.0 / 86400), (2, 3.0 / 86400))


def span_pulsars(spans=OWN_SPANS, seed=0):
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, (n, span) in enumerate(spans):
        t0 = rng.uniform(53000.0, 58800.0 - span)
        mjd = np.sort(t0 + np.r_[0.0, span, rng.uniform(0, span, n - 2)])
        ra, dec = rng.uniform(0, 24), math.degrees(math.asin(rng.uniform(-1, 1)))
        p = pulsar_from_arrays(f"S{j:03d}", {"RAJ": float(ra), "DECJ": float(dec)}, mjd.astype(np.longdouble),
                               rng.uniform(0.3, 3.0, n), flags=[{"f": "A"}] * n)
        make_ideal(p)
        out.append(p)
    return out


def fourier_batch(kind, K, conv, plan_only=False):
    """"gen": the generator edge batch (one frequency grid); "own": ``span_pulsars`` with each pulsar's default
    Tspan (different frequencies per pulsar)."""
    from tests import generator_reference as GR
    if kind == "gen":
        return GR.gen_batch(red=K, conv=conv, white=False, ecorr=False, plan_only=plan_only)
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(span_pulsars(), plan_only=plan_only)
    for i in range(b.n_psr):
        b.set_red(i, -13.8, 3.5, components=K, libstempo_convention=conv)
    return b


# ------------------------------------------------------------------ catalogs and sweeps
def catalog(n_src, seed=0, merged=0.1, los=False):
    """A random catalog [8, n_src] (gwtheta, gwphi, mc [Msun], dist [Mpc], fgw [Hz], phase0, psi, inc): fgw 1e-9 ..
    1e-6, mc 1e8 .. 1e10; a fraction ``merged`` of heavy, fast binaries that merge before or inside the span; ``los``:
    source 0 at gwtheta = 0 (on the line of sight of a pulsar at dec +90 deg)."""
    rng = np.random.default_rng(seed)
    cat = np.stack([np.arccos(rng.uniform(-1, 1, n_src)), rng.uniform(0, 2 * np.pi, n_src), 10 ** rng.uniform(8, 10, n_src),
                    10 ** rng.uniform(1, 3, n_src), 10 ** rng.uniform(-9, -6, n_src), rng.uniform(0, 2 * np.pi, n_src),
                    rng.uniform(0, np.pi, n_src), np.arccos(rng.uniform(-1, 1, n_src))])
    m = rng.uniform(size=n_src) < merged
    cat[2, m] = 10 ** rng.uniform(9.5, 10, m.sum())
    cat[4, m] = 10 ** rng.uniform(-7.5, -6.5, m.sum())
    if los:
        cat[0, 0] = 0.0
    return np.ascontiguousarray(cat)


def merger_margin(pre, t):
    """min over sources and TOAs (Earth and pulsar term) of |1 - fac1 t|: a catalog whose margin exceeds 1e-9 has
    an unambiguous set of NaN (merged) sources."""
    fac1, cm, pd = pre[:, 1:2], pre[:, 12:13], pre[:, 13:14]
    with np.errstate(invalid="ignore"):
        tp = t[None, :] - pd * (1 - cm)
        m = np.minimum(np.abs(1 - fac1 * t[None, :]), np.abs(1 - fac1 * tp))
    return float(np.nanmin(m)) if np.isfinite(m).any() else np.inf


def phat_of(ra, dec):
    """add_catalog_of_cws' pulsar direction from (RA, DEC) [rad]."""
    ptheta, pphi = np.pi / 2 - dec, ra
    return (float(np.sin(ptheta) * np.cos(pphi)), float(np.sin(ptheta) * np.sin(pphi)), float(np.cos(ptheta)))


def auto_slices(n_src):
    """The slice count add_catalog_of_cws chooses."""
    return int(max(1, min(64, (n_src + 255) // 256)))


CW_TOAS, CW_STAGE = 128, 32
# (n_src, n_slices ("auto" or a count, "n+5": empty slices), n_toa, CAT_VARIANTS branch, accumulate)
CAT_CASES = (
    (1, "auto", 1, "evolve", 0), (1, "n+5", 129, "pphase", 1), (31, "auto", 127, "earth", 0), (31, 3, 128, "approx", 1),
    (32, "auto", 129, "mono", 0), (32, 64, 1025, "evolve", 0), (33, "auto", 128, "pphase", 0), (33, 3, 127, "earth", 1),
    (256, "auto", 1025, "approx", 0), (256, 3, 1, "mono", 0), (257, "auto", 129, "evolve", 1), (257, 64, 128, "earth", 0),
    (4097, "auto", 1025, "mono", 0), (4097, "n+5", 129, "approx", 0), (16385, "auto", 1025, "evolve", 0),
    (16385, 1, 127, "pphase", 1), (16385, "n+5", 128, "earth", 0))


def n_slices_of(n_src, spec):
    return auto_slices(n_src) if spec == "auto" else (n_src + 5 if spec == "n+5" else int(spec))


def slice_lengths(n_src, n_slices):
    per = -(-n_src // n_slices)
    return [max(0, min(n_src, (k + 1) * per) - k * per) for k in range(n_slices)]


def cat_variant(tag):
    """(mode, psr_term, pdist, pphase, use_pphase) of a CAT_VARIANTS branch."""
    from tests.test_oracle_pinning import CAT_VARIANTS
    v = CAT_VARIANTS[tag]
    mode = 0 if v.get("evolve", True) else (1 if v.get("phase_approx", False) else 2)
    pph = v.get("pphase")
    return mode, int(v.get("psrTerm", True)), float(v.get("pdist", 1.0)), float(pph or 0.0), int(pph is not None)


def toa_sample(n_toa, n_src, rng, budget=300_000, m=40):
    """TOA indices the catalog reference evaluates: all of them when n_src n_toa is small, else ~``m`` including each
    CTA's first and last TOA."""
    if n_src * n_toa <= budget:
        return np.arange(n_toa)
    edges = np.unique(np.r_[np.arange(0, n_toa, CW_TOAS), np.minimum(np.arange(CW_TOAS - 1, n_toa + CW_TOAS - 1, CW_TOAS), n_toa - 1)])
    extra = rng.choice(n_toa, size=max(0, m - len(edges)), replace=False)
    return np.unique(np.r_[edges, extra])


def cat_toas(n_toa, seed=0, tref=53000 * 86400.0):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.sort(rng.uniform(53000.0, 58800.0, n_toa)) * 86400.0 - tref)


# CGW sources of the det sweep: (gwtheta, gwphi, mc, dist, fgw, phase0, psi, inc, tref [s]); the near-merger source is
# added per batch (``near_merger``)
CGW_SOURCES = (
    (0.0, 1.0, 1e8, 10.0, 1e-9, 0.3, 0.2, 0.0, 0.0),
    (np.pi, 2.0, 1e9, 50.0, 1e-8, 1.1, 1.3, np.pi / 2, 53000 * 86400.0),
    (1.2, 4.0, 1e10, 300.0, 1e-8, 2.0, 2.9, np.pi, 53000 * 86400.0),
    (1.9, 3.3, 3e8, 30.0, 1e-7, 2.2, 0.4, 0.0, 53000 * 86400.0),
    (2.3, 5.5, 1e8, 100.0, 1e-6, 4.0, 0.7, 1.0, 58800 * 86400.0),      # would merge inside the span with an earlier tref
    (0.7, 0.3, 1e10, 1000.0, 1e-9, 5.9, 0.1, np.pi / 2, 0.0),
)


def near_merger(mjd_all, mc=1e9, fgw=5e-8, margin=1e-6):
    """A CGW source (tuple as CGW_SOURCES) that merges just after the last TOA: tref puts the last TOA at 1 - margin of
    the time to merger (1 - fac1 t = margin there)."""
    mc_s, w0 = mc * SOLAR2S, np.pi * fgw
    fac1 = 256 / 5 * mc_s ** (5 / 3) * w0 ** (8 / 3)
    tref = float(np.max(mjd_all)) * 86400 - (1 - margin) / fac1
    return (1.0, 2.0, mc, 20.0, fgw, 0.4, 0.9, 0.8, tref)
