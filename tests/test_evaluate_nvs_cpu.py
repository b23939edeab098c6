"""CPU: the host pieces of the novel-view evaluation -- the quaternion of a rotation matrix that renders at a
ground-truth pose use, and which test views `evaluate_nvs` scores."""
import pytest
import torch

from splatam_b200 import mapping as M
from splatam_b200.evaluate import evaluate_nvs, select_nvs_frames


def test_matrix_to_quaternion_inverts_build_rotation():
    g = torch.Generator().manual_seed(4)
    q = torch.nn.functional.normalize(torch.randn(64, 4, generator=g, dtype=torch.float64), dim=1)
    # each component in turn the largest, and the 180-degree rotations where w = 0
    q = torch.cat([q, torch.eye(4, dtype=torch.float64), torch.tensor([[0.0, 0.6, 0.8, 0.0]], dtype=torch.float64)])
    for qi, R in zip(q, M.build_rotation(q)):
        got = M.matrix_to_quaternion(R)
        sign = 1.0 if float((got * qi).sum()) >= 0 else -1.0      # q and -q are the same rotation
        assert torch.allclose(got * sign, qi, atol=1e-12), (qi, got)
    w2c = torch.eye(4)
    w2c[:3, :3] = M.build_rotation(q[:1].float())[0]
    w2c[:3, 3] = torch.tensor([0.1, -0.2, 0.3])
    pose, quat = M.gt_pose(w2c)
    assert pose is w2c and quat.shape == (1, 4) and abs(float(quat.norm()) - 1) < 1e-6


def test_nvs_frame_selection_skips_the_train_frame():
    assert select_nvs_frames(6, 1) == [1, 2, 3, 4, 5]
    assert select_nvs_frames(6, 2) == [1, 2, 4]              # test views k = 0, 1, 3
    assert select_nvs_frames(12, 5) == [1, 5, 10]
    assert select_nvs_frames(1, 1) == []


def test_no_cpu_fallback():
    params = dict(means3D=torch.zeros(2, 3))
    with pytest.raises(Exception, match="CUDA"):
        evaluate_nvs(params, [dict(im=torch.zeros(3, 200, 200))], None, 0.5, 0, False)
