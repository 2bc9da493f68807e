"""`-m gpu`: the sm_90a build of kb_core.h / kb_aff.h (tests/probe/libkbprobe.so, device = 1) against the same Python references and
cases as tests/test_core_arith.py checks the host build with.  The device code differs from the host code where it matters:
div_0_to_10 estimates with __fdividef (MUFU.RCP), the doubles go through __dsub_rn / __ddiv_rn / __dmul_rn / __double2ll_rz."""
import pytest

import test_core_arith as A

pytestmark = pytest.mark.gpu


def test_div_0_to_10_device_build_is_exact():
    A.check_div(1)


def test_least_and_most_requested_device_build():
    A.check_requested(1)


def test_balanced_score_device_build():
    A.check_balanced(1)


def test_le_func_and_res_less_equal_device_build():
    A.check_le(1)


def test_affinity_scores_device_build():
    A.check_aff(1)


@pytest.mark.parametrize("geometry,R,W", A.EVAL_GEOMETRIES)
def test_eval_pair_device_build(geometry, R, W):
    A.check_eval_pair(1, geometry, R, W)
