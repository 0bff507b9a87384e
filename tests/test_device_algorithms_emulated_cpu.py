"""NumPy model of a device code path that has not run on a GPU yet (DESIGN.md section 9), kept as a CPU test so that
the claim "index maps checked by emulation" stays reproducible:

* psd_small_kernel, d.triangle == 2 -- load / store index maps of the real embedding of a Hermitian matrix.

The functions below follow the CUDA code statement by statement (same scalars, same tests, same order)."""
import math

import numpy as np

from oracle import cosmo_oracle as O


def _svec_pos(i, j):
    return j * (j + 1) // 2 + i


def kernel_load_complex(x, Nc):
    """psd_small_kernel, load branch d.triangle == 2"""
    N, inv = 2 * Nc, 1.0 / math.sqrt(2.0)
    M = np.zeros((N, N))
    for j in range(N):
        for i in range(N):
            I, bi, J, bj = i % Nc, i // Nc, j % Nc, j // Nc
            a, b = (I, J) if I < J else (J, I)
            if bi == bj:
                v = x[_svec_pos(a, b)]
                if a != b:
                    v *= inv
            elif I == J:
                v = 0.0
            else:
                im_ab = x[Nc * (Nc + 1) // 2 + b * (b - 1) // 2 + a] * inv
                b_IJ = im_ab if I < J else -im_ab
                v = b_IJ if bi == 1 else -b_IJ
            M[i, j] = v
    return M


def kernel_store_complex(V, Nc):
    """psd_small_kernel, store branch d.triangle == 2 (V already scaled by sqrt(max(lambda, 0)))"""
    N, tri, sqrt2 = 2 * Nc, Nc * (Nc + 1) // 2, math.sqrt(2.0)
    s = np.zeros(Nc * Nc)
    for e in range(Nc * Nc):
        imag = e >= tri
        ee = e - tri if imag else e
        if not imag:
            j = int((math.sqrt(8.0 * ee + 1.0) - 1.0) * 0.5)
            while (j + 1) * (j + 2) // 2 <= ee:
                j += 1
            while j * (j + 1) // 2 > ee:
                j -= 1
            i = ee - j * (j + 1) // 2
            acc = 0.5 * sum(V[i, k] * V[j, k] + V[Nc + i, k] * V[Nc + j, k] for k in range(N))
            s[e] = acc if i == j else sqrt2 * acc
        else:
            j = int((math.sqrt(8.0 * ee + 1.0) + 1.0) * 0.5)
            while j * (j + 1) // 2 <= ee:
                j += 1
            while j * (j - 1) // 2 > ee:
                j -= 1
            i = ee - j * (j - 1) // 2
            acc = sum(V[Nc + i, k] * V[j, k] - V[i, k] * V[Nc + j, k] for k in range(N))
            s[e] = sqrt2 * 0.5 * acc
    return s


def test_complex_psd_embedding_index_maps():
    rng = np.random.default_rng(4)
    for Nc in (2, 3, 7):
        Z = rng.standard_normal((Nc, Nc)) + 1j * rng.standard_normal((Nc, Nc))
        X = (Z + Z.conj().T) / 2
        x = O.extract_upper_triangle_complex(X, math.sqrt(2.0))
        M = kernel_load_complex(x, Nc)
        assert np.allclose(M, np.block([[X.real, -X.imag], [X.imag, X.real]]), atol=1e-15)
        w, Q = np.linalg.eigh(M)
        s = kernel_store_complex(Q * np.sqrt(np.maximum(w, 0)), Nc)
        ref = x.copy()
        O.project_cone(ref, O.ComplexPsdConeTriangle(Nc * Nc))
        assert np.max(np.abs(s - ref)) < 1e-13
