"""The OPQ restatement (tests/opq_reference.py) checked without a GPU: the random start against the C++ standard
library it restates, the Procrustes contract against numpy and against wrong rotations, and the host SVD the engine
solves each round with (vearch_b200/csrc/jacobi_svd.h) on the rank-deficient X^T Y a constant dimension produces."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import opq_reference as orf
from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vearch_b200", "csrc")
CXX = shutil.which("g++") or shutil.which("c++")
needs_cxx = pytest.mark.skipif(CXX is None, reason="no C++ compiler")

START_SRC = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
int main(int argc, char** argv) {
  const int d = atoi(argv[1]);
  std::vector<double> R((size_t)d * d);
  std::mt19937 rng(1234);
  std::normal_distribution<double> nd(0.0, 1.0);
  for (auto& v : R) v = nd(rng);
  for (int i = 0; i < d; i++) {
    for (int p = 0; p < i; p++) {
      double dot = 0;
      for (int j = 0; j < d; j++) dot += R[(size_t)i * d + j] * R[(size_t)p * d + j];
      for (int j = 0; j < d; j++) R[(size_t)i * d + j] -= dot * R[(size_t)p * d + j];
    }
    double nrm = 0;
    for (int j = 0; j < d; j++) nrm += R[(size_t)i * d + j] * R[(size_t)i * d + j];
    nrm = sqrt(nrm);
    for (int j = 0; j < d; j++) R[(size_t)i * d + j] /= nrm;
  }
  fwrite(R.data(), 8, R.size(), stdout);
}
"""

SVD_SRC = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "jacobi_svd.h"
int main(int argc, char** argv) {  // reads d, then a d x d matrix (fp64), writes R = V U^T as the OPQ round forms it
  int d;
  if (fread(&d, 4, 1, stdin) != 1) return 1;
  std::vector<double> a((size_t)d * d), U, V, R((size_t)d * d);
  if (fread(a.data(), 8, a.size(), stdin) != a.size()) return 1;
  gb::jacobi_svd(a, d, d, &U, &V);
  for (int i = 0; i < d; i++)
    for (int j = 0; j < d; j++) {
      double acc = 0;
      for (int k = 0; k < d; k++) acc += V[(size_t)i * d + k] * U[(size_t)j * d + k];
      R[(size_t)i * d + j] = acc;
    }
  fwrite(R.data(), 8, R.size(), stdout);
}
"""


def compile_cxx(tmp_path, name, src):
    """the program built the way the engine's host code is (g++ -O3, no -march: no FMA contraction)"""
    c = tmp_path / f"{name}.cc"
    c.write_text(src)
    exe = tmp_path / name
    subprocess.check_call([CXX, "-O3", "-std=c++17", "-I", CSRC, str(c), "-o", str(exe)])
    return str(exe)


# ---- the random start ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1234, 5, 2 ** 32 - 1])
def test_mt19937_drives_rand_perm(seed):
    """the Python MT19937 draws what the oracle's std::mt19937 draws: its Fisher-Yates gives orc.rand_perm"""
    n = 3000
    g = orf.MT19937(seed)
    perm = np.arange(n)
    for i in range(n - 1):
        j = i + g() % (n - i)
        perm[i], perm[j] = perm[j], perm[i]
    assert np.array_equal(perm, orc.rand_perm(n, seed))


@needs_cxx
@pytest.mark.parametrize("d", [1, 2, 8, 30, 64, 128])
def test_random_start_matches_libstdcxx(tmp_path, d):
    exe = compile_cxx(tmp_path, "start", START_SRC)
    want = np.frombuffer(subprocess.check_output([exe, str(d)]), np.float64).reshape(d, d)
    got = orf.random_start(d)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert np.abs(got @ got.T - np.eye(d)).max() < 1e-13


# ---- the Procrustes contract ------------------------------------------------------------------------------------------
def procrustes_np(A):
    u, _, vt = np.linalg.svd(A)
    return vt.T @ u.T


def test_procrustes_contract_accepts_numpy_and_rejects_wrong_rotations():
    rng = np.random.default_rng(1)
    A = rng.standard_normal((16, 16))
    R = procrustes_np(A)
    assert orf.check_procrustes(R, A) is None
    assert "orthonormal" in orf.check_procrustes(R * (1 + 1e-9), A)
    q, _ = np.linalg.qr(rng.standard_normal((16, 16)))
    assert "optimal" in orf.check_procrustes(q, A)
    # the optimum has a single-sign freedom per zero singular value: the contract accepts either, numpy or not
    A[3] = 0
    R = procrustes_np(A)
    u, s, vt = np.linalg.svd(A)
    flip = vt.T @ np.diag(np.r_[np.ones(15), -1.0]) @ u.T
    assert orf.check_procrustes(R, A) is None and orf.check_procrustes(flip, A) is None


def test_mean_contract():
    rng = np.random.default_rng(2)
    xs = (rng.standard_normal((5000, 6)) * 100 + 1000).astype(np.float32)
    exact = xs.astype(np.float64).mean(0).astype(np.float32)
    assert orf.check_mean(exact, xs) is None
    assert orf.check_mean(np.nextafter(np.nextafter(exact, np.inf), np.inf), xs) is not None


# ---- the host SVD -----------------------------------------------------------------------------------------------------
def rank_deficient(kind, d, rng):
    A = rng.standard_normal((d, d))
    if kind == "zero_row":
        A[5] = 0
    elif kind == "zero_rows8":
        A[rng.choice(d, 8, replace=False)] = 0
    elif kind == "zero_cols8":
        A[:, rng.choice(d, 8, replace=False)] = 0
    elif kind == "low_rank":
        A = rng.standard_normal((d, 7)) @ rng.standard_normal((7, d))
    elif kind == "zero":
        A[:] = 0
    elif kind == "tiny_row":  # a column of U with a norm near the rounding noise of the others
        A[2] = 1e-290
    return A


@needs_cxx
@pytest.mark.parametrize("kind", ["full", "zero_row", "zero_rows8", "zero_cols8", "low_rank", "zero", "tiny_row"])
@pytest.mark.parametrize("d", [8, 64])
def test_jacobi_svd_rotation_is_orthonormal_and_optimal(tmp_path, kind, d):
    """R = V U^T from the engine's SVD is orthonormal to 1e-12 and maximises trace(R A), whatever the rank of A (a
    constant training dimension makes a row of X^T Y exactly 0)"""
    exe = compile_cxx(tmp_path, "svd", SVD_SRC)
    A = rank_deficient(kind, d, np.random.default_rng(d))
    out = subprocess.run([exe], input=np.int32(d).tobytes() + A.astype(np.float64).tobytes(), capture_output=True,
                         check=True).stdout
    R = np.frombuffer(out, np.float64).reshape(d, d)
    r = orf.check_procrustes(R, A)
    assert r is None, r
