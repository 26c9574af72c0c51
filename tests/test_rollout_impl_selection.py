"""rollout.fused_kernel -> the rollout implementation RolloutWorker runs (select_rollout_impl), on the host: the `auto`
thresholds (tensor-core kernel from TC_AUTO_MIN_ENVS environments, SIMT kernel up to FUSED_AUTO_MAX_ENVS_PER_CTA
environments per SM), chunked policies, unsupported shapes and the two configuration errors."""
import pytest

from rlinf_b200.rollout import FUSED_AUTO_MAX_ENVS_PER_CTA, TC_AUTO_MIN_ENVS, select_rollout_impl


def test_thresholds():
    assert (TC_AUTO_MIN_ENVS, FUSED_AUTO_MAX_ENVS_PER_CTA) == (640, 16)


@pytest.mark.parametrize("fused_kernel,C,B,sms,tc_ok,simt_ok,impl", [
    # auto, C = 1: tensor-core kernel from 640 environments on, where it supports the shapes
    ("auto", 1, 640, 132, True, True, "tc"),
    ("auto", 1, 4096, 132, True, True, "tc"),
    ("auto", 1, 639, 132, True, True, "simt"),
    # below 640 or outside the tensor-core envelope: SIMT kernel up to 16 environments per SM (16 x 132 = 2112)
    ("auto", 1, 2112, 132, False, True, "simt"),
    ("auto", 1, 2113, 132, False, True, "graph"),
    ("auto", 1, 128, 8, False, True, "simt"),
    ("auto", 1, 129, 8, False, True, "graph"),
    ("auto", 1, 256, 132, True, False, "graph"),
    ("auto", 1, 4096, 132, False, False, "graph"),
    # auto, C > 1: the per-kernel loop at every size
    ("auto", 4, 256, 132, True, False, "graph"),
    ("auto", 4, 4096, 132, True, False, "graph"),
    ("auto", 4, 4096, 132, False, False, "graph"),
    # tc: the tensor-core kernel at any size it supports
    ("tc", 1, 64, 132, True, True, "tc"),
    ("tc", 4, 64, 132, True, False, "tc"),
    ("tc", 8, 4096, 132, True, False, "tc"),
    # simt / True: the SIMT kernel where it supports the shapes, else the per-kernel loop
    ("simt", 1, 4096, 132, True, True, "simt"),
    (True, 1, 64, 132, True, True, "simt"),
    (True, 1, 5000, 132, True, False, "graph"),
    # False: the per-kernel loop
    (False, 1, 4096, 132, True, True, "graph"),
    (False, 4, 4096, 132, True, False, "graph"),
])
def test_select_rollout_impl(fused_kernel, C, B, sms, tc_ok, simt_ok, impl):
    assert select_rollout_impl(fused_kernel, C, B, sms, tc_ok, simt_ok) == impl


@pytest.mark.parametrize("fused_kernel", ["simt", True])
def test_simt_with_chunks_raises(fused_kernel):
    with pytest.raises(ValueError, match="SIMT rollout kernel implements num_action_chunks == 1"):
        select_rollout_impl(fused_kernel, 2, 1024, 132, True, False)


@pytest.mark.parametrize("C,msg", [(1, "needs hidden 256, a value head, act_dim <= 8"),
                                   (4, "with num_action_chunks > 1 needs hidden 256")])
def test_tc_outside_envelope_raises(C, msg):
    with pytest.raises(ValueError, match=msg):
        select_rollout_impl("tc", C, 1024, 132, False, C == 1)
