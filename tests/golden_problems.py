"""Literal problem data copied *as data* from the reference's own tests/examples
(SURVEY.md section 8c, G1..G14).  Each builder returns ``(P, q, constraints)``
in the reference's user-facing form (A x + b in K) using oracle cone classes;
``expected`` holds the reference's known answers and tolerances.
"""
import numpy as np
import scipy.sparse as sp

from oracle import cosmo_oracle as O


def g1_qp_nonneg():
    """examples/qp.jl:13-27 — x*=[0.3,0.7], obj=1.88 (tol 1e-3)."""
    q = np.array([1.0, 1.0])
    P = np.array([[4.0, 1.0], [1.0, 2.0]])
    A = np.array([[1.0, 1.0], [1.0, 0.0], [0.0, 1.0]])
    l = np.array([1.0, 0.0, 0.0])
    u = np.array([1.0, 0.7, 0.7])
    Aa = np.vstack([-A, A])
    ba = np.concatenate([u, -l])
    return P, q, [O.Constraint(Aa, ba, O.Nonnegatives(6))]


def g1_qp_box():
    """examples/qp.jl:31-35."""
    q = np.array([1.0, 1.0])
    P = np.array([[4.0, 1.0], [1.0, 2.0]])
    A = np.array([[1.0, 1.0], [1.0, 0.0], [0.0, 1.0]])
    l = np.array([1.0, 0.0, 0.0])
    u = np.array([1.0, 0.7, 0.7])
    return P, q, [O.Constraint(A, np.zeros(3), O.Box(l, u))]


G1_X = np.array([0.3, 0.7])
G1_OBJ = 1.88


def g2_box_feasible():
    """test/UnitTests/qp-box.jl:15-32 — Solved, obj=-0.5 (atol 1e-5)."""
    A = np.eye(2)
    return np.eye(2), np.array([1.0, -1.0]), [O.Constraint(A, np.zeros(2), O.Box([0.0, 0.0], [1.0, 1.0]))]


def g2_box_primal_infeasible_1():
    """qp-box.jl:35-52 — Primal_infeasible."""
    A = np.array([[1.0, 0.0], [1.0, 0.0]])
    return np.eye(2), np.array([1.0, -1.0]), [O.Constraint(A, np.array([2.0, 0.0]), O.Box([0.0, 0.0], [1.0, 1.0]))]


def g2_box_primal_infeasible_2():
    """qp-box.jl:54-71 — Primal_infeasible."""
    A = np.array([[1.0, 0.0], [1.0, 0.0]])
    return np.eye(2), np.array([1.0, -1.0]), [O.Constraint(A, np.zeros(2), O.Box([0.0, 2.0], [1.0, 3.0]))]


def g2_box_dual_infeasible():
    """qp-box.jl:73-106 — Dual_infeasible (scaling=0/check_infeasibility=20 and scaling=10/40)."""
    A = np.eye(2)
    return np.zeros((2, 2)), np.array([1.0, 1.0]), [O.Constraint(A, np.ones(2), O.Box([0.0, -np.inf], [1.0, 3.0]))]


def g12_lp():
    """examples/lp.jl:17-46 — x*=[3,5,1,1], obj=20 (atol 1e-2); eps_abs=1e-4, eps_rel=1e-5."""
    c = np.array([1.0, 2.0, 3.0, 4.0])
    n = 4
    I = np.eye(4)
    c1 = O.Constraint(-I, 10.0 * np.ones(4), O.Nonnegatives(4))
    c2 = O.Constraint(I, -np.ones(4), O.Nonnegatives(4))
    A3 = np.zeros((1, n)); A3[0, 1] = 1.0          # Constraint(1, -5, Nonnegatives, n, 2:2)
    c3 = O.Constraint(A3, np.array([-5.0]), O.Nonnegatives(1))
    c4 = O.Constraint(np.array([[1.0, 0.0, 1.0, 0.0]]), np.array([-4.0]), O.Nonnegatives(1))
    return np.zeros((4, 4)), c, [c1, c2, c3, c4]


G12_X = np.array([3.0, 5.0, 1.0, 1.0])
G12_OBJ = 20.0


def svec_index(i, j):
    """0-based position of (i,j), i<=j, in the column-major upper triangle (convexset.jl:432-442)."""
    return j * (j + 1) // 2 + i


def g13_lovasz_petersen():
    """examples/lovasz_petersen.jl:22-60 — theta(Petersen) = 4.

    JuMP form: max sum(X) s.t. tr X = 1, X_ij = 0 on edges, X PSD.  Restated in
    COSMO's native svec form: variable x = svec(X) (off-diagonals * sqrt2),
    min -<J, X> = -(sum_diag x + sqrt2 * sum_offdiag x).
    """
    n = 10
    edges = [(1, 2), (1, 5), (1, 6), (2, 3), (2, 7), (3, 4), (3, 8), (4, 5), (4, 9), (5, 10),
             (6, 8), (6, 9), (7, 9), (7, 10), (8, 10)]
    d = n * (n + 1) // 2
    q = np.zeros(d)
    for j in range(n):
        for i in range(j + 1):
            q[svec_index(i, j)] = -1.0 if i == j else -np.sqrt(2.0)
    rows = [np.zeros(d)]
    for j in range(n):
        rows[0][svec_index(j, j)] = 1.0
    bz = [-1.0]
    for (a, b) in edges:
        r = np.zeros(d)
        r[svec_index(a - 1, b - 1)] = 1.0
        rows.append(r)
        bz.append(0.0)
    Az = np.vstack(rows)
    cz = O.Constraint(Az, np.array(bz), O.ZeroSet(len(bz)))
    cp = O.Constraint(sp.identity(d, format="csr"), np.zeros(d), O.PsdConeTriangle(d))
    return np.zeros((d, d)), q, [cz, cp]


G13_OBJ = -4.0


def g3_hs21():
    """test/UnitTests/moi_wrapper.jl:219-276 — HS21 (Maros-Meszaros) with redundant
    constraints added in unsorted order to exercise set merging / sorting.
    Known answers: obj = -99.96 (= 0.5 x'Px + r, r = -100), x = [-2, 0]; set order
    Zero / Nonneg / Box / SOC.  Restated through the native Constraint form
    (A x + b in K) instead of MOI."""
    P = np.diag([0.02, 2.0])
    q = np.zeros(2)
    A = np.array([[-10.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])
    x_true = np.array([-2.0, 0.0])
    nn1 = O.Constraint(A[0:1, :], np.array([-10.0]), O.Nonnegatives(1))            # A1 x >= 10
    soc = O.Constraint(np.array([[-1.0, 0.0], [0.0, 1.0]]), np.zeros(2), O.SecondOrderCone(2))
    box1 = O.Constraint(A[1:2, :], np.zeros(1), O.Box([2.0], [50.0]))
    zero1 = O.Constraint(np.array([[1.0, 0.0]]), np.array([2.0]), O.ZeroSet(1))      # x1 == -2
    nn2 = O.Constraint(-np.eye(2), 10.0 * np.ones(2), O.Nonnegatives(2))            # x - 10 <= 0
    box2 = O.Constraint(A[2:3, :], np.zeros(1), O.Box([-50.0], [50.0]))
    zeroset = O.Constraint(np.eye(2), -x_true, O.ZeroSet(2))
    return P, q, [nn1, soc, box1, zero1, nn2, box2, zeroset]


G3_X = np.array([-2.0, 0.0])
G3_OBJ = -99.96 + 100.0  # the constant r = -100 is carried outside the solver


def g14_update_qp():
    """test/UnitTests/model_modifications.jl:33-47: G1 then update!(q=[2,3]) -> obj 3.5? (x=[0.5,0.5])."""
    return g1_qp_nonneg()


# ---------------------------------------------------------------------------
# G15 / G16: exponential and power cone problems (test/UnitTests/exp_cone.jl, pow_cone.jl)
# Each entry: (name, builder, expected status, expected objective or None, atol, settings)
# ---------------------------------------------------------------------------
_I3 = np.eye(3)
_Z3 = np.zeros((3, 3))
_E5 = float(np.exp(5.0))


def g15_exp_feasible():
    """exp_cone.jl:19-43 — max x s.t. y e^(x/y) <= z, y = 1, z = e^5: Solved, obj = -5 (atol 1e-2)."""
    return _Z3, np.array([-1.0, 0, 0]), [O.Constraint(_I3, np.zeros(3), O.ExponentialCone()),
                                         O.Constraint([[0, 1.0, 0], [0, 0, 1.0]], [-1.0, -_E5], O.ZeroSet(2))]


def g15_exp_primal_infeasible_1():
    """exp_cone.jl:47-77 — y = 1, z = -1: Primal_infeasible."""
    return _Z3, np.array([1.0, 0, 0]), [O.Constraint(_I3, np.zeros(3), O.ExponentialCone()),
                                        O.Constraint([[0, -1.0, 0]], [-1.0], O.ZeroSet(1)),
                                        O.Constraint([[0, 0, -1.0]], [1.0], O.ZeroSet(1))]


def g15_exp_primal_infeasible_2():
    """exp_cone.jl:79-104 — two shifted cones that cannot intersect: Primal_infeasible."""
    return _Z3, np.array([1.0, 0, 0]), [O.Constraint(_I3, [0, 0, -0.2], O.ExponentialCone()),
                                        O.Constraint(-_I3, [0, 0, -0.3], O.ExponentialCone())]


def g15_exp_dual_infeasible():
    """exp_cone.jl:106-124 — max z over the cone: Dual_infeasible."""
    return _Z3, np.array([0, 0, -1.0]), [O.Constraint(_I3, np.zeros(3), O.ExponentialCone())]


def g15_dualexp_feasible():
    """exp_cone.jl:130-156 — min y s.t. -x e^(y/x) <= e z, x = -1, z = e^5: Solved, obj = -6 (atol 1e-3)."""
    return _Z3, np.array([0, 1.0, 0]), [O.Constraint(_I3, np.zeros(3), O.DualExponentialCone()),
                                        O.Constraint([[1.0, 0, 0], [0, 0, 1.0]], [1.0, -_E5], O.ZeroSet(2))]


def g15_dualexp_primal_infeasible():
    """exp_cone.jl:160-185 — u = 1 violates u <= 0 of the dual cone: Primal_infeasible."""
    return _Z3, np.ones(3), [O.Constraint(_I3, np.zeros(3), O.DualExponentialCone()),
                             O.Constraint([[1.0, 0, 0], [0, 1.0, 0]], [-1.0, -2.0], O.ZeroSet(2))]


def g16_pow_feasible():
    """pow_cone.jl:16-56 — max x1^0.6 y^0.4 + x2^0.1: Solved, obj = -1.8458 (atol 1e-3), max_iter = 5000."""
    q = np.zeros(6)
    q[2] = q[5] = -1.0
    A1 = np.zeros((3, 6)); A1[:, 0:3] = _I3
    A2 = np.zeros((3, 6)); A2[:, 3:6] = _I3
    return np.zeros((6, 6)), q, [O.Constraint(A1, np.zeros(3), O.PowerCone(0.6)),
                                 O.Constraint(A2, np.zeros(3), O.PowerCone(0.1)),
                                 O.Constraint([[1.0, 2.0, 0, 3.0, 0, 0]], [-3.0], O.ZeroSet(1)),
                                 O.Constraint([[0, 0, 0, 0, 1.0, 0]], [-1.0], O.ZeroSet(1))]


def g16_pow_primal_infeasible():
    """pow_cone.jl:77-95 — x = y = 1, z = 2: Primal_infeasible."""
    return _Z3, np.array([0, 0, -1.0]), [O.Constraint(_I3, np.zeros(3), O.PowerCone(0.8)),
                                         O.Constraint(_I3, [-1.0, -1.0, -2.0], O.ZeroSet(3))]


def g16_pow_dual_infeasible():
    """pow_cone.jl:97-111 — min z over the cone: Dual_infeasible."""
    return _Z3, np.array([0, 0, 1.0]), [O.Constraint(_I3, np.zeros(3), O.PowerCone(0.8))]


def g16_dualpow_feasible():
    """pow_cone.jl:116-137 — max z s.t. (x/.8)^.8 (y/.2)^.2 >= z, x = .8, y = .2: Solved, obj = -1 (atol 1e-3)."""
    return _Z3, np.array([0, 0, -1.0]), [O.Constraint(_I3, np.zeros(3), O.DualPowerCone(0.8)),
                                         O.Constraint([[1.0, 0, 0], [0, 1.0, 0]], [-0.8, -0.2], O.ZeroSet(2))]


G15_G16 = [
    ("exp_feasible", g15_exp_feasible, "Solved", -5.0, 1e-2, dict(eps_abs=1e-4, eps_rel=1e-4)),
    ("exp_primal_infeasible_1", g15_exp_primal_infeasible_1, "Primal_infeasible", None, None, {}),
    ("exp_primal_infeasible_2", g15_exp_primal_infeasible_2, "Primal_infeasible", None, None, {}),
    ("exp_dual_infeasible", g15_exp_dual_infeasible, "Dual_infeasible", None, None, {}),
    ("dualexp_feasible", g15_dualexp_feasible, "Solved", -6.0, 1e-3, {}),
    ("dualexp_primal_infeasible", g15_dualexp_primal_infeasible, "Primal_infeasible", None, None, {}),
    ("pow_feasible", g16_pow_feasible, "Solved", -1.8458, 1e-3, dict(max_iter=5000)),
    ("pow_primal_infeasible", g16_pow_primal_infeasible, "Primal_infeasible", None, None, {}),
    ("pow_dual_infeasible", g16_pow_dual_infeasible, "Dual_infeasible", None, None, {}),
    ("dualpow_feasible", g16_dualpow_feasible, "Solved", -1.0, 1e-3, {}),
]


# ---------------------------------------------------------------------------
# G4 / G5 / G6 / G11 (SURVEY.md 8c)
# ---------------------------------------------------------------------------
def _svec_scale(N):
    """diagonal of the map 'unscaled upper triangle (MOI) -> svec' (sqrt 2 on off-diagonal entries)"""
    out = []
    for j in range(N):
        for i in range(j + 1):
            out.append(1.0 if i == j else np.sqrt(2.0))
    return np.array(out)


def g4_small_sdp():
    """test/UnitTests/moi_wrapper.jl:39-106 — min <C,X> s.t. <A1,X> = 11, <A2,X> = 19, X PSD (3x3), x = upper
    triangle of X by columns; the test asserts the two constraint primals (11, 19 at atol 1e-3)."""
    A1_t = np.array([1.0, 0, 3, 2, 14, 5])
    A2_t = np.array([0.0, 4, 6, 16, 0, 4])
    C_t = np.array([1.0, 4, 9, 6, 0, 7])
    cons = [O.Constraint(A1_t[None, :], [-11.0], O.ZeroSet(1)), O.Constraint(A2_t[None, :], [-19.0], O.ZeroSet(1)),
            O.Constraint(np.diag(_svec_scale(3)), np.zeros(6), O.PsdConeTriangle(6))]
    return np.zeros((6, 6)), C_t, cons


G4_A1 = np.array([1.0, 0, 3, 2, 14, 5])
G4_A2 = np.array([0.0, 4, 6, 16, 0, 4])


def g5_sigma_max_lmi():
    """test/UnitTests/nuclear_norm_minimization.jl:16-41 — min t s.t. [tI Y; Y' tI] PSD (PsdConeTriangle(21)),
    Y[2,1] <= 4, Y[2,2] >= 3, sum(Y) >= 12; x = [t; vec(Y)].  Expected: t = sigma_max(Y) (1e-3)."""
    q = np.concatenate([[1.0], np.zeros(9)])
    c1 = np.zeros((1, 10)); c1[0, 2] = -1.0
    c2 = np.zeros((1, 10)); c2[0, 5] = 1.0
    c3 = np.concatenate([[0.0], np.ones(9)])[None, :]
    A_lmi = np.zeros((21, 10))
    for r in (0, 2, 5, 9, 14, 20):                       # diagonal entries of the 6x6 matrix
        A_lmi[r, 0] = -1.0
    for col, r in enumerate((6, 7, 8, 10, 11, 12, 15, 16, 17)):   # rows 7,8,9,11,12,13,16,17,18 (1-based)
        A_lmi[r, 1 + col] = -np.sqrt(2.0)
    cons = [O.Constraint(c1, [4.0], O.Nonnegatives(1)), O.Constraint(c2, [-3.0], O.Nonnegatives(1)),
            O.Constraint(c3, [-12.0], O.Nonnegatives(1)), O.Constraint(-A_lmi, np.zeros(21), O.PsdConeTriangle(21))]
    return np.zeros((10, 10)), q, cons


def g6_chordal_sdp_data():
    """examples/chordal_decomposition.jl:7-10 — min c'x s.t. B - A1 x1 - A2 x2 PSD (9x9, common sparsity pattern)."""
    A1 = np.array([[-4.0, 0, -2, 0, 0, -1, 0, 0, 0], [0, -3, -1, 0, 0, 0, 0, 0, 0], [-2, -1, -2, 0, 0, 5, 4, -4, 0],
                   [0, 0, 0, -4, -5, 0, 0, 3, 0], [0, 0, 0, -5, 4, 0, 0, 2, 0], [-1, 0, 5, 0, 0, 5, -4, -4, -5],
                   [0, 0, 4, 0, 0, -4, -1, -1, -3], [0, 0, -4, 3, 2, -4, -1, 2, -2], [0, 0, 0, 0, 0, -5, -3, -2, -3]])
    A2 = np.array([[-5.0, 0, 3, 0, 0, -2, 0, 0, 0], [0, -3, -5, 0, 0, 0, 0, 0, 0], [3, -5, 3, 0, 0, 5, -4, -5, 0],
                   [0, 0, 0, 3, 2, 0, 0, -2, 0], [0, 0, 0, 2, 4, 0, 0, -3, 0], [-2, 0, 5, 0, 0, 1, -5, -2, -4],
                   [0, 0, -4, 0, 0, -5, -2, -3, 3], [0, 0, -5, -2, -3, -2, -3, 5, 3], [0, 0, 0, 0, 0, -4, 3, 3, -4]])
    B = np.array([[-0.11477375644968069, 0, 6.739182490600791, 0, 0, -1.2185593245043502, 0, 0, 0],
                  [0, 1.2827680528587497, -5.136452036888789, 0, 0, 0, 0, 0, 0],
                  [6.739182490600791, -5.136452036888789, 7.344770673489607, 0, 0, -0.2224400187044442, -10.505300166831221,
                   -1.2627361794562273, 0],
                  [0, 0, 0, 10.327710040060499, 8.91534585379813, 0, 0, -6.525873789637007, 0],
                  [0, 0, 0, 8.91534585379813, 0.8370459338528677, 0, 0, -6.210900615408826, 0],
                  [-1.2185593245043502, 0, -0.2224400187044442, 0, 0, -3.8185953011245024, -0.994033914192722,
                   2.8156077981712997, 1.4524716674219218],
                  [0, 0, -10.505300166831221, 0, 0, -0.994033914192722, 0.029162208619863517, -2.8123790276830745,
                   7.663416446183705],
                  [0, 0, -1.2627361794562273, -6.525873789637007, -6.210900615408826, 2.8156077981712997,
                   -2.8123790276830745, 4.71893305728242, 6.322431630550857],
                  [0, 0, 0, 0, 0, 1.4524716674219218, 7.663416446183705, 6.322431630550857, 0.5026094532322212]])
    c = np.array([-0.21052661285686525, -1.263324575834677])
    return A1, A2, B, c


def _svec(M):
    N = M.shape[0]
    out = []
    for j in range(N):
        for i in range(j + 1):
            out.append(M[i, j] if i == j else np.sqrt(2.0) * M[i, j])
    return np.array(out)


def g6_chordal_sdp():
    """the same problem as a PsdConeTriangle(45) constraint  svec(B) - svec(A1) x1 - svec(A2) x2 in K."""
    A1, A2, B, c = g6_chordal_sdp_data()
    A = -np.column_stack([_svec(A1), _svec(A2)])
    return np.zeros((2, 2)), c, [O.Constraint(A, _svec(B), O.PsdConeTriangle(45))]


G6_CLIQUES = [[0, 2, 5], [1, 2], [2, 5, 6, 7], [3, 4, 7], [5, 6, 7, 8]]   # docs/src/decomposition.md:43 (0-based)


def g11_iteration_limit():
    """test/UnitTests/moi_wrapper.jl:201-217 — max x s.t. x >= 10 with max_iter = 2: Max_iter_reached,
    rho_updates == [0.1]."""
    return np.zeros((1, 1)), np.array([-1.0]), [O.Constraint([[1.0]], [-10.0], O.Nonnegatives(1))]


def g17_complex_least_eigenvalue():
    """test/UnitTests/least_eigenvalue.jl:8-39 — min <C, X> s.t. tr X = 1, X Hermitian PSD, for
    C = [1 i 0; -i 1 i; 0 -i 1]: the least eigenvalue 1 - sqrt 2 (atol = rtol = 1e-4); PsdConeTriangle{T, Complex{T}}(9)."""
    C = np.array([[1, 1j, 0], [-1j, 1, 1j], [0, -1j, 1]])
    d = 3
    vec_c = O.extract_upper_triangle_complex(C, np.sqrt(2.0))
    id_vec = np.zeros(d * d)
    for k in range(1, d + 1):
        id_vec[k * (k + 1) // 2 - 1] = 1.0
    cons = [O.Constraint(id_vec[None, :], [-1.0], O.ZeroSet(1)),
            O.Constraint(np.eye(d * d), np.zeros(d * d), O.ComplexPsdConeTriangle(d * d))]
    return np.zeros((d * d, d * d)), vec_c, cons


G17_OBJ = 1.0 - np.sqrt(2.0)


# ---------------------------------------------------------------------------
# Infeasible problems of test/UnitTests/InfeasibilityTests/ (primal_infeasible_1/2/3, dual_infeasible_1/2).
# The reference draws its data from MersenneTwister streams that cannot be reproduced here, so these builders follow
# the construction of each file (sizes, sparsity, the feasible or unbounded part and the row that breaks it) with
# numpy's generator and a fixed seed.  The seeds are ones for which the CPU oracle (EmptyAccelerator and
# AndersonAccelerator, scaling 0 and 10) reaches the status the reference's file asserts.
# ---------------------------------------------------------------------------
def _sprand(rng, m, n, density):
    """sprand(rng, m, n, density): uniform [0, 1) values at a Bernoulli pattern"""
    mask = rng.random((m, n)) < density
    return sp.csr_matrix(np.where(mask, rng.random((m, n)), 0.0))


def _pos_def(rng, n, a_min=0.1, a_max=2.0):
    """generate_pos_def_matrix (COSMOTestUtils.jl:11-19): Q diag(eigs) Q' with eigs uniform in [a_min, a_max]"""
    Q, _ = np.linalg.qr(rng.random((n, n)))
    X = (Q * (rng.random(n) * (a_max - a_min) + a_min)) @ Q.T
    return 0.5 * (X + X.T)


def _svec_upper(X):
    """the PsdConeTriangle vector of a symmetric matrix (upper triangle by columns, sqrt 2 off the diagonal)"""
    N = X.shape[0]
    return np.concatenate([np.concatenate([X[:j, j] * np.sqrt(2.0), [X[j, j]]]) for j in range(N)])


def primal_infeasible_1(seed=74747):
    """primal_infeasible_1.jl: x >= 0, A >= 0, b < 0, s in R+ (one Nonnegatives constraint)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(5, 51))
    m = 2 * n
    A = sp.vstack([_sprand(rng, m, n, 0.8), -sp.identity(n)]).tocsr()
    b = np.concatenate([-rng.random(m), np.zeros(n)])
    P = _pos_def(rng, n)
    ytrue, xtrue = rng.random(m + n), rng.random(n)
    q = -P @ xtrue - A.T @ ytrue
    return P, q, [O.Constraint(-A, b, O.Nonnegatives(m + n))]


def primal_infeasible_2(seed=29, r=None, triangle=False, m1=None):
    """primal_infeasible_2.jl: ZeroSet rows with a feasible right-hand side, x >= 0, and a PsdCone whose constant part
    is entrywise negative (A >= 0, x >= 0: the diagonal is negative).  The PSD rows of A are arbitrary, so delta_y is not
    symmetric on the square cone.  triangle=True: the same with a PsdConeTriangle; r: the side (r >= 97 for the large
    path); m1: the number of ZeroSet rows (the reference uses r^2)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(10, 51))
    r = int(rng.integers(2, 11)) if r is None else r
    m2 = r * (r + 1) // 2 if triangle else r * r
    m1 = m2 if m1 is None else m1
    A = _sprand(rng, m1 + m2, n, 0.8) * 50
    xtrue = rng.random(n) * 50
    b1 = A[:m1] @ xtrue
    b3 = -rng.random(m2)
    P = _pos_def(rng, n)
    Afull = sp.vstack([A[:m1], -sp.identity(n), A[m1:]]).tocsr()
    Y3 = _pos_def(rng, r)
    ytrue = np.concatenate([rng.standard_normal(m1) * 50, rng.random(n) * 50,
                            _svec_upper(Y3) if triangle else Y3.reshape(-1, order="F")])
    q = -P @ xtrue - Afull.T @ ytrue
    cone = O.PsdConeTriangle(m2) if triangle else O.PsdCone(m2)
    return P, q, [O.Constraint(-A[:m1], b1, O.ZeroSet(m1)), O.Constraint(sp.identity(n), np.zeros(n), O.Nonnegatives(n)),
                  O.Constraint(-A[m1:], b3, cone)]


def primal_infeasible_3(seed=1313, psd=True):
    """primal_infeasible_3.jl: ZeroSet + SecondOrderCone + PsdCone around a feasible point, then the SOC's first row is
    replaced by 0 x + (-1): t = -1 < 0.  The reference accepts Primal_infeasible or Max_iter_reached.
    psd=False: the SOC-only variant (ZeroSet + SecondOrderCone)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(10, 51))
    m1, m2, r = int(rng.integers(2, 11)), int(rng.integers(3, 11)), int(rng.integers(4, 11))
    m3 = r * r if psd else 0
    A = (_sprand(rng, m1 + m2 + m3, n, 0.8) * 50).tolil()
    xtrue = rng.random(n) * 50
    s = np.concatenate([np.zeros(m1), rng.random(m2), _pos_def(rng, r).reshape(-1, order="F") if psd else []])
    b = A @ xtrue + s
    A[m1, :] = 0
    b[m1] = -1.0
    A = A.tocsr()
    P = _pos_def(rng, n)
    y2 = rng.random(m2 - 1) * 50
    ytrue = np.concatenate([rng.random(m1) * 50, [np.linalg.norm(y2) + 1.0], y2,
                            _pos_def(rng, r, 0.1, 5.0).reshape(-1, order="F") if psd else []])
    q = -P @ xtrue - A.T @ ytrue
    cons = [O.Constraint(-A[:m1], b[:m1], O.ZeroSet(m1)), O.Constraint(-A[m1:m1 + m2], b[m1:m1 + m2], O.SecondOrderCone(m2))]
    if psd:
        cons.append(O.Constraint(-A[m1 + m2:], b[m1 + m2:], O.PsdCone(m3)))
    return P, q, cons


def dual_infeasible_1(seed=1):
    """dual_infeasible_1.jl: the last variable has cost -1 and appears in no constraint (P = 0)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(5, 51))
    m = 2 * n
    A = (_sprand(rng, m, n, 0.7) * 50).tolil()
    A[:, n - 1] = 0
    A = A.tocsr()
    q = rng.random(n) * 50
    q[-1] = -1.0
    b = A @ (rng.random(n) * 50) + rng.random(m) * 50
    return sp.csr_matrix((n, n)), q, [O.Constraint(-A, b, O.Nonnegatives(m))]


def dual_infeasible_2(seed=8):
    """dual_infeasible_2.jl: ZeroSet + Nonnegatives + SecondOrderCone + PsdCone around a feasible point, x1 unbounded
    below (cost -1, in no row but the Nonnegatives row x1 >= ... that lets it decrease)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(10, 51))
    m1, m2, m3, r = int(rng.integers(2, 11)), 1, int(rng.integers(3, 11)), int(rng.integers(4, 11))
    m4 = r * r
    A = (_sprand(rng, m1 + m2 + m3 + m4, n, 0.8) * 50).tolil()
    xtrue = rng.random(n) * 50
    s3 = rng.random(m3 - 1)
    s = np.concatenate([np.zeros(m1), [rng.random()], [np.linalg.norm(s3) + 1.0], s3, _pos_def(rng, r).reshape(-1, order="F")])
    A[:, 0] = 0
    A[m1, :] = 0
    A[m1, 0] = -1.0
    A = A.tocsr()
    b = A @ xtrue + s
    b[m1] = 0.0
    q = np.concatenate([[-1.0], rng.random(n - 1)])
    o = np.cumsum([0, m1, m2, m3, m4])
    return sp.csr_matrix((n, n)), q, [O.Constraint(-A[o[0]:o[1]], b[o[0]:o[1]], O.ZeroSet(m1)),
                                      O.Constraint(-A[o[1]:o[2]], b[o[1]:o[2]], O.Nonnegatives(m2)),
                                      O.Constraint(-A[o[2]:o[3]], b[o[2]:o[3]], O.SecondOrderCone(m3)),
                                      O.Constraint(-A[o[3]:o[4]], b[o[3]:o[4]], O.PsdCone(m4))]


# (name, builder, statuses the reference's file accepts)
INFEASIBILITY_PROBLEMS = [
    ("primal_infeasible_1", primal_infeasible_1, ("Primal_infeasible",)),
    ("primal_infeasible_2", primal_infeasible_2, ("Primal_infeasible",)),
    ("primal_infeasible_2_triangle", lambda: primal_infeasible_2(seed=2024, triangle=True), ("Primal_infeasible",)),
    # N = 100 > 96: the block-Jacobi certificate.  The oracle detects it with EmptyAccelerator only (with
    # AndersonAccelerator it reaches max_iter on every seed tried), so the solve tests run it without acceleration
    ("primal_infeasible_2_large_psd", lambda: primal_infeasible_2(seed=97, r=100, triangle=True, m1=20), ("Primal_infeasible",)),
    ("primal_infeasible_3", primal_infeasible_3, ("Primal_infeasible", "Max_iter_reached")),
    ("primal_infeasible_3_soc", lambda: primal_infeasible_3(psd=False), ("Primal_infeasible", "Max_iter_reached")),
    ("dual_infeasible_1", dual_infeasible_1, ("Dual_infeasible",)),
    ("dual_infeasible_2", dual_infeasible_2, ("Dual_infeasible",)),
]
