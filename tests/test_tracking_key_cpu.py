"""CPU: the key a captured tracking iteration is cached under (mapping._tracking_key) names the storage of every
Gaussian tensor the iteration reads, so a map with one tensor swapped for another of the same shape never replays a
graph captured over the old one."""
import torch

from splatam_b200 import mapping as M


def test_tracking_key_names_every_gaussian_tensor():
    P = 64
    gauss = dict(means3D=torch.rand(P, 3), rgb_colors=torch.rand(P, 3), unnorm_rotations=torch.rand(P, 4),
                 logit_opacities=torch.rand(P, 1), log_scales=torch.rand(P, 1))
    frame = dict(id=1, cam=object(), im=torch.rand(3, 8, 8))
    args = (20, 0.0004, 0.002, None)
    key = M._tracking_key(gauss, frame, *args)
    assert M._tracking_key({k: v.detach() for k, v in gauss.items()}, dict(frame), *args) == key
    for k in M.GAUSSIAN_KEYS:
        assert M._tracking_key(dict(gauss, **{k: torch.rand_like(gauss[k])}), frame, *args) != key, k
