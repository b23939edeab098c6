"""CPU: LPIPS weight loading and packing (evaluate.LpipsAlex), the feature sizes of the float64 oracle
(oracle/lpips_torch.py), argument checks of the sb_lpips entry points before any launch, and no CPU fallback."""
import ctypes

import pytest
import torch

from oracle import lpips_torch as OL
from splatam_b200 import _lib
from splatam_b200 import evaluate as EV

CONVS = ((0, 3, 64, 11), (3, 64, 192, 5), (6, 192, 384, 3), (8, 384, 256, 3), (10, 256, 256, 3))


def _write(tmp_path, alex, lin):
    a, b = tmp_path / "alexnet-owt-7be5be79.pth", tmp_path / "alex.pth"
    torch.save(alex, a)
    torch.save(lin, b)
    return str(a), str(b)


def test_load_packs_both_state_dicts(tmp_path):
    alex, lin = OL.random_state_dicts(seed=1)
    net = EV.LpipsAlex.load(*_write(tmp_path, alex, lin), device="cpu")
    w = net.weights
    assert w.dtype == torch.float32 and w.device.type == "cpu"
    assert w.numel() == _lib.nbytes("sb_lpips_weights_floats")
    off = 0
    for idx, cin, cout, k in CONVS:                 # [K][Cout], then the bias
        K = cin * k * k
        got = w[off:off + K * cout].reshape(K, cout)
        assert torch.equal(got, alex["features.%d.weight" % idx].reshape(cout, K).t())
        off += K * cout
        assert torch.equal(w[off:off + cout], alex["features.%d.bias" % idx])
        off += cout
    for l, (_, _, cout, _) in enumerate(CONVS):
        assert torch.equal(w[off:off + cout], lin["lin%d.model.1.weight" % l].reshape(-1))
        off += cout
    assert off == w.numel()
    # classifier keys are ignored: dropping them packs the same buffer
    no_cls = {k: v for k, v in alex.items() if not k.startswith("classifier.")}
    assert torch.equal(EV.LpipsAlex.from_state_dicts(no_cls, lin, "cpu").weights, w)


@pytest.mark.parametrize("which,key", [("alex", "features.6.weight"), ("alex", "features.10.bias"),
                                       ("lin", "lin3.model.1.weight")])
def test_missing_key_or_bad_shape_raises_naming_the_key(tmp_path, which, key):
    alex, lin = OL.random_state_dicts(seed=2)
    sd = alex if which == "alex" else lin
    good = sd[key]
    del sd[key]
    with pytest.raises(_lib.SplatamB200Error, match="missing key '%s'" % key.replace(".", r"\.")):
        EV.LpipsAlex.load(*_write(tmp_path, alex, lin), device="cpu")
    sd[key] = good[:, :-1] if good.dim() == 4 else good[:-1]
    with pytest.raises(_lib.SplatamB200Error, match=key.replace(".", r"\.") + ".*has shape"):
        EV.LpipsAlex.load(*_write(tmp_path, alex, lin), device="cpu")


def test_oracle_feature_sizes():
    alex, lin = OL.random_state_dicts(seed=0)
    weights = dict(alex, **lin)
    for (H, W), want in (((680, 1200), [(169, 299), (84, 149), (41, 74), (41, 74), (41, 74)]),
                         ((31, 31), [(7, 7), (3, 3), (1, 1), (1, 1), (1, 1)])):
        x = torch.empty(2, 3, H, W, device="meta")
        fs = OL.features(x, weights, dtype=torch.float32)
        assert [tuple(f.shape[-2:]) for f in fs] == want
        assert [f.shape[1] for f in fs] == [64, 192, 384, 256, 256] and all(f.shape[0] == 2 for f in fs)
    x = torch.rand(1, 3, 31, 31, generator=torch.Generator().manual_seed(0))
    assert torch.equal(OL.lpips(x, x.clone(), weights), torch.zeros(1, dtype=torch.float64))
    assert float(OL.lpips(x, 1 - x, weights)[0]) > 0


def test_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_lpips_weights_floats(ctypes.byref(n)) == 0 and n.value == 2_470_848
    assert lib.sb_lpips_weights_floats(None) == 1
    assert lib.sb_lpips_workspace_bytes(1, 680, 1200, ctypes.byref(n)) == 0
    one = n.value
    assert 77e6 < one < 80e6                  # ~39 MB of activations per image, and a pair runs two images
    assert lib.sb_lpips_workspace_bytes(2, 680, 1200, ctypes.byref(n)) == 0 and n.value > 1.9 * one
    assert lib.sb_lpips_workspace_bytes(1, 31, 31, ctypes.byref(n)) == 0 and n.value > 0
    for N, H, W in ((0, 64, 64), (-1, 64, 64), (1, 30, 64), (1, 64, 30), (1, -5, 64)):
        assert lib.sb_lpips_workspace_bytes(N, H, W, ctypes.byref(n)) == 1, (N, H, W)
    assert lib.sb_lpips_workspace_bytes(1, 64, 64, None) == 1
    assert lib.sb_lpips_workspace_bytes(1, 64, 64, ctypes.byref(n)) == 0
    need, big = n.value, 1 << 34
    # non-null dummy pointers are never dereferenced: every check comes before the first CUDA call
    assert lib.sb_lpips(None, 1, 1, 64, 64, 1, 1, big, 1, 1, None) == 1
    assert lib.sb_lpips(1, None, 1, 64, 64, 1, 1, big, 1, 1, None) == 1
    assert lib.sb_lpips(1, 1, 1, 64, 64, None, 1, big, 1, 1, None) == 1                  # no weights
    assert lib.sb_lpips(1, 1, 1, 64, 64, 1, None, big, 1, 1, None) == 1                  # no workspace
    assert lib.sb_lpips(1, 1, 1, 64, 64, 1, 1, big, None, None, None) == 1               # nowhere to write
    assert lib.sb_lpips(1, 1, 0, 64, 64, 1, 1, big, 1, 1, None) == 1                     # N < 1
    assert lib.sb_lpips(1, 1, 1, 30, 64, 1, 1, big, 1, 1, None) == 1                     # H < 31
    assert lib.sb_lpips(1, 1, 1, 64, 30, 1, 1, big, 1, None, None) == 1                  # W < 31
    assert lib.sb_lpips(1, 1, 1, 64, 64, 1, 1, need - 1, 1, None, None) == 2             # SB_ERR_WORKSPACE


def test_no_cpu_fallback():
    alex, lin = OL.random_state_dicts(seed=0)
    net = EV.LpipsAlex.from_state_dicts(alex, lin, "cpu")
    x = torch.rand(1, 3, 64, 64)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        EV.lpips(x, x, net)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        EV.lpips(x, x, net, size_average=False)
