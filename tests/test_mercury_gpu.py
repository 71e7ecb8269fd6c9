"""The Mercury entry points (b200_mat_vec_rows, b200_div_binomial, b200_mercury_s_poly) bit-exact against the
oracle, the device prover (nova_b200.mercury) field for field against oracle/mercury_ref.py, accepted by the
restated verifier at benchmark-like sizes of both parities, and snark / ppsnark with ee="mercury"."""
import pytest

import mercury_parity as mp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sp(b200):
    from nova_b200 import spartan
    return spartan


@pytest.mark.parametrize("cols", [1, 2, 1 << 11])
@pytest.mark.parametrize("rows", [1, 2, 63, 64, 65, 1 << 10, 1 << 11])
def test_div_binomial(sp, oracle, rows, cols):
    mp.check_div_binomial(sp, oracle, rows, cols)


@pytest.mark.parametrize("rows,cols", [(1, 1), (2, 3), (65, 2), (1 << 11, 1 << 11), (600000, 1), (1 << 20, 2)])
def test_div_binomial_zero_and_last_row(sp, oracle, rows, cols):
    """zero polynomials, and only the last row non-zero: the carry crosses every chunk (and, for 600000 or
    2^20 rows, both levels of the suffix scan)"""
    for kind in ("zero", "last_row"):
        mp.check_div_binomial(sp, oracle, rows, cols, kind)


def test_div_binomial_two_level_random(sp, oracle):
    mp.check_div_binomial(sp, oracle, 600000, 1)


@pytest.mark.parametrize("rows,cols", [(1, 1), (3, 5), (64, 2048), (2048, 2048), (1024, 2048)])
def test_mat_vec_rows(sp, oracle, rows, cols):
    mp.check_mat_vec_rows(sp, oracle, rows, cols)


@pytest.mark.parametrize("b", [2, 4, 1 << 11, 1 << 12])
def test_s_poly(sp, oracle, b):
    mp.check_s_poly(sp, oracle, b)


@pytest.mark.parametrize("ell", [2, 3, 10, 15, 16])
def test_mercury_prove_matches_oracle(b200, oracle, ell):
    mp.run_prove(b200, oracle, ell)


@pytest.mark.parametrize("ell", [20, 21])
def test_mercury_proof_verifies_at_scale(b200, oracle, ell):
    mp.run_verify_only(b200, oracle, ell)


def test_snark_with_mercury(b200, oracle):
    mp.run_snark(b200, oracle)


def test_ppsnark_with_mercury(b200, oracle):
    mp.run_ppsnark(b200, oracle)
