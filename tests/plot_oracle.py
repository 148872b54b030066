"""Host reference for the KR balancing the contact-map tests compare against: bnewt (Knight & Ruiz, IMA J. Numer. Anal.
33(3), 2013), restated in numpy with the step limits and the step counts the device path reports."""

import numpy as np


class NotConverged(RuntimeError):
    pass


def bnewt(A, tol=1e-6, delta=0.1, Delta=3, max_outer=1000, max_inner=10000):
    """(x, outer steps, inner CG steps) balancing the symmetric matrix A: diag(x) A diag(x) has unit row sums."""
    n = A.shape[0]
    e = np.ones(n)
    g, etamax = 0.9, 0.1
    eta = etamax
    stop_tol = tol * 0.5
    x = e.copy()
    rt = tol ** 2
    v = x * (A @ x)
    rk = 1 - v
    rho_km1 = rk @ rk
    rout = rold = rho_km1
    outer = inner = 0
    while rout > rt:
        outer += 1
        if outer > max_outer:
            raise NotConverged("outer")
        k, mm = 0, 0
        y = e.copy()
        innertol = max(eta ** 2 * rout, rt)
        while rho_km1 > innertol:
            mm += 1
            if mm > max_inner:
                raise NotConverged("inner")
            k += 1
            if k == 1:
                Z = rk / v
                p = Z
                rho_km1 = rk @ Z
            else:
                p = Z + (rho_km1 / rho_km2) * p
            w = x * (A @ (x * p)) + v * p
            alpha = rho_km1 / (p @ w)
            ap = alpha * p
            ynew = y + ap
            if ynew.min() <= delta:
                ind = ap < 0
                y = y + ((delta - y[ind]) / ap[ind]).min() * ap
                break
            if ynew.max() >= Delta:
                ind = ynew > Delta
                y = y + ((Delta - y[ind]) / ap[ind]).min() * ap
                break
            y = ynew
            rk = rk - alpha * w
            rho_km2 = rho_km1
            Z = rk / v
            rho_km1 = rk @ Z
        x = x * y
        v = x * (A @ x)
        rk = 1 - v
        rho_km1 = rk @ rk
        rout = rho_km1
        inner += k
        rat = rout / rold
        rold = rout
        eta_o = eta
        eta = g * rat
        if g * eta_o ** 2 > 0.1:
            eta = max(eta, g * eta_o ** 2)
        eta = max(min(eta, etamax), stop_tol / np.sqrt(rout))
    return x, outer, inner
