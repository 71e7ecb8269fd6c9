"""The ppsnark + IPA composition of the oracle's pieces (ppsnark_ipa_ref.prove_ipa: prove_core, then ipa_prove on the
batched claim, ipa_pc.rs:64-77) passes the restated verifier (ppsnark_ipa_ref.verify_ipa: verify_core, the batched commitment and
ipa_verify, ipa_pc.rs:80-100) on all four curves, and an altered eval_W, L_vec[0] or a_hat fails."""
import pytest

import spark_ipa_parity as sip
import ppsnark_ipa_ref as ipr
from oracle.pyref import CURVES


@pytest.mark.parametrize("cid", [0, 1, 2, 3])
def test_prove_ipa_verifies(cid):
    c = CURVES[cid]
    p = c.q
    inst = sip.instance(cid)
    S = inst["S"]

    def verify(proof):
        return ipr.verify_ipa(p, c, inst["ck_pts"], inst["ck_c"], S["num_cons"], S["num_vars"], inst["N"], inst["U"],
                             inst["S_comm"], 909, proof)
    ref = inst["ref"]
    assert verify(ref)
    L_vec, R_vec, a_hat = ref["eval_arg"]
    assert len(L_vec) == len(R_vec) == inst["N"].bit_length() - 1
    assert not verify(dict(ref, eval_W=(ref["eval_W"] + 1) % p))
    assert not verify(dict(ref, eval_arg=([c.add(L_vec[0], c.gen)] + list(L_vec[1:]), R_vec, a_hat)))
    assert not verify(dict(ref, eval_arg=(L_vec, R_vec, (a_hat + 1) % p)))


def test_ipa_verify_with_a_given_msm_agrees():
    """a given `msm` only replaces how the verifier's N-point MSM (ck_hat) is computed"""
    c = CURVES[1]
    p = c.q
    inst = sip.instance(1)
    S = inst["S"]
    calls = []

    def msm(s, pts):
        calls.append(len(pts))
        return c.msm_naive(s, pts)
    assert ipr.verify_ipa(p, c, inst["ck_pts"], inst["ck_c"], S["num_cons"], S["num_vars"], inst["N"], inst["U"],
                         inst["S_comm"], 909, inst["ref"], msm=msm)
    assert calls == [inst["N"]]
