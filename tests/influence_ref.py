"""float64 restatement of calculate_diagnostics_gpu (diagnostics.c:620-1182, influence_function.cu of the
reference), index for index as the reference's kernels read and write, for the tests of
tests/test_cpu_diagnostics.py and tests/test_gpu_diagnostics.py.

Rows are n = t*Nbase + b.  coh and res: [R][4] complex (XX, XY, YX, YY) of channel 0; p: the Jones
[nchunk][N][8] of one cluster; the chunk of row n is n // ceil(R / nchunk).  Complex matrices are
numpy arrays indexed [row, col]."""
import numpy as np


def jones(p, N, nchunk, R, sta):
    """[R][2][2] Jones of station sta[n] at row n, from the row's hybrid chunk"""
    per = (R + nchunk - 1) // nchunk
    chunk = np.arange(R) // per
    pj = np.asarray(p, dtype=np.float64).reshape(nchunk, N, 4, 2)
    J = pj[chunk, sta, :, 0] + 1j * pj[chunk, sta, :, 1]
    return J.reshape(R, 2, 2)


def kron2(A, B):
    """batched kron of 2x2 matrices: [n][4][4], [2a+c][2b+d] = A[a,b] B[c,d]"""
    return np.einsum("nab,ncd->nacbd", A, B).reshape(-1, 4, 4)


def _tr(A):
    return np.swapaxes(A, -1, -2)


def hessian(N, Nbase, T, sta1, sta2, flag, p, nchunk, coh, res):
    """kernel_hessian: the 4N x 4N Hessian of one cluster over the unflagged rows, before the
    conditioning.  A thread adds K[off, i] at (row 4*rowsta + i, col 4*colsta + off), i.e. K^T"""
    R = Nbase * T
    C = np.asarray(coh).reshape(R, 2, 2)
    Rs = np.asarray(res).reshape(R, 2, 2)
    Jp = jones(p, N, nchunk, R, sta1)
    Jq = jones(p, N, nchunk, R, sta2)
    I2 = np.broadcast_to(np.eye(2), (R, 2, 2))
    K_qp = kron2(-_tr(C), np.conj(_tr(Rs)))                # -C^T (x) R^H -> (q, p)
    A = C @ np.conj(_tr(Jq))
    K_pp = kron2(_tr(A @ np.conj(_tr(A))), I2)              # D^T (x) I2, D = (C Jq^H)(C Jq^H)^H
    K_pq = kron2(-np.conj(C), Rs)                           # -conj(C) (x) R -> (p, q)
    B = Jp @ C
    K_qq = kron2(_tr(np.conj(_tr(B)) @ B), I2)              # D^T (x) I2, D = (Jp C)^H (Jp C)
    H = np.zeros((4 * N, 4 * N), dtype=np.complex128)
    ok = np.flatnonzero(np.asarray(flag) == 0)
    ii = np.arange(4)
    for K, rs, cs in ((K_qp, sta2, sta1), (K_pp, sta1, sta1), (K_pq, sta1, sta2), (K_qq, sta2, sta2)):
        rows = 4 * np.asarray(rs)[ok][:, None, None] + ii[None, :, None]
        cols = 4 * np.asarray(cs)[ok][:, None, None] + ii[None, None, :]
        np.add.at(H, (rows, cols), _tr(K[ok]))
    return H


def adv(N, Nbase, T, sta1, sta2, flag, p, nchunk, coh):
    """kernel_d_solutions: 4N x Nbase, split station layout (rows 2p+{0,1}, 2N+2p+{0,1}); column
    n % Nbase gets, per unflagged row, H [1+j, 1+j, 1+j, 1+j] with H read row major from
    kron(conj(C) J_q^T, I2) stored column major"""
    R = Nbase * T
    C = np.asarray(coh).reshape(R, 2, 2)
    Jq = jones(p, N, nchunk, R, sta2)
    K = kron2(np.conj(C) @ _tr(Jq), np.broadcast_to(np.eye(2), (R, 2, 2)))
    Hrm = _tr(K)                       # the row-major reading of a column-major array
    prod = Hrm.sum(axis=2) * (1 + 1j)  # [R][4]
    out = np.zeros((4 * N, Nbase), dtype=np.complex128)
    ok = np.flatnonzero(np.asarray(flag) == 0)
    bl = ok % Nbase
    s1 = np.asarray(sta1)[ok]
    for r in range(2):
        np.add.at(out, (2 * s1 + r, bl), prod[ok, r])
        np.add.at(out, (2 * N + 2 * s1 + r, bl), prod[ok, r + 2])
    return out


def d_residuals(N, Nbase, T, sta1, sta2, p, nchunk, coh, X):
    """kernel_d_residuals: [4][Nbase][Nbase], EVERY row (no flag test); row n adds, to row n % Nbase
    of every column bl, H x with H the row-major reading of kron(conj(J_q) C^T, I2) and x the
    split-layout rows of station sta1 in column bl of X (4N x Nbase)"""
    R = Nbase * T
    C = np.asarray(coh).reshape(R, 2, 2)
    Jq = jones(p, N, nchunk, R, sta2)
    K = kron2(np.conj(Jq) @ _tr(C), np.broadcast_to(np.eye(2), (R, 2, 2)))
    Hrm = _tr(K)
    dR = np.zeros((4, Nbase, Nbase), dtype=np.complex128)
    for t in range(T):   # one timeslot at a time: [Nbase][4][Nbase] per step
        sl = slice(t * Nbase, (t + 1) * Nbase)
        s1 = np.asarray(sta1)[sl]
        Jv = np.stack([X[2 * s1], X[2 * s1 + 1], X[2 * N + 2 * s1], X[2 * N + 2 * s1 + 1]], axis=1)
        dR += np.transpose(np.einsum("nij,njb->nib", Hrm[sl], Jv), (1, 0, 2))
    return dR


def condition(H, hadd=0.0):
    """diagnostics.c:711-751: abs() of C on a float is the integer abs, so every real diagonal entry
    that truncates to 0 (|h| < 1) becomes 1; then + hadd on every real diagonal entry"""
    H = H.copy()
    d = np.real(np.diag(H)).copy()
    d = np.where(np.trunc(d) == 0, 1.0, d) + hadd
    H[np.diag_indices_from(H)] = d + 1j * np.imag(np.diag(H))
    return H


def consensus_hadd(rho_k, Bpoly, Bi_k):
    """0.5 rho Fd1, Fd = 1 - Bpoly^T Bi Bpoly (Bi column major), Fd1 = Fd^2 (1 + Fd^2 / (1 - Fd^2))"""
    Bi_k = np.asarray(Bi_k).reshape(len(Bpoly), len(Bpoly)).T
    Fd = 1.0 - Bpoly @ (Bi_k @ Bpoly)
    Fdd = Fd * Fd
    return 0.5 * rho_k * Fdd * (1.0 + Fdd / (1.0 - Fdd))


def eig_to_x(E, Nbase, T):
    """find_eigenvalues' layout: E[c] the Nbase eigenvalues of correlation c; their interleaved
    doubles e; x[8b+2c] = e[b], x[8b+2c+1] = e[Nbase+b] in timeslot 0, copied to every timeslot.
    returns channel 0 of x, [T*Nbase*8]"""
    x0 = np.zeros(8 * Nbase)
    for c in range(4):
        e = np.empty(2 * Nbase)
        e[0::2] = np.real(E[c])
        e[1::2] = np.imag(E[c])
        x0[2 * c::8] = e[:Nbase]
        x0[2 * c + 1::8] = e[Nbase:]
    return np.tile(x0, T)


def x_to_eig(x0, Nbase):
    """the inverse of eig_to_x on timeslot 0: the four correlations' eigenvalues"""
    E = []
    for c in range(4):
        e = np.concatenate([x0[2 * c:8 * Nbase:8], x0[2 * c + 1:8 * Nbase:8]])
        E.append(e[0::2] + 1j * e[1::2])
    return E


def diagnostics(N, Nbase, T, sta1, sta2, flag, clusters, res, hadd=None):
    """steps 2-5 over clusters: each a dict(p, nchunk, coh); returns (dR, [H conditioned], [X])"""
    dR = np.zeros((4, Nbase, Nbase), dtype=np.complex128)
    Hs, Xs = [], []
    for k, c in enumerate(clusters):
        H = condition(hessian(N, Nbase, T, sta1, sta2, flag, c["p"], c["nchunk"], c["coh"], res),
                      0.0 if hadd is None else hadd[k])
        A = adv(N, Nbase, T, sta1, sta2, flag, c["p"], c["nchunk"], c["coh"])
        X = np.linalg.solve(H, A)
        dR += d_residuals(N, Nbase, T, sta1, sta2, c["p"], c["nchunk"], c["coh"], X)
        Hs.append(H)
        Xs.append(X)
    return dR, Hs, Xs
