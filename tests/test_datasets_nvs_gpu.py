"""GPU: the ScanNet++ and ReplicaV2 readers (splatam_b200/datasets.py) through the ingest kernel against the
reference's own dataset classes (tests/golden/datasets/ref_nvs_datasets.npz): colour and depth bit for bit for every
read of both splits -- ScanNet++'s JPEG colour at the exact-2x and a non-2x size, ReplicaV2's PNG colour natively and
downscaled -- with the synchronous and the prefetching reader."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from util import GOLDEN
from splatam_b200 import datasets as D

pytestmark = pytest.mark.gpu

FIX = os.path.join(GOLDEN, "datasets", "ref_nvs_datasets.npz")
READS = ["scannetpp_train", "scannetpp_train_bad", "scannetpp_test", "scannetpp_test_bad", "replicav2_train",
         "replicav2_test", "replicav2_test_sel"]


@pytest.fixture(scope="module")
def gen():
    spec = importlib.util.spec_from_file_location("make_golden_nvs_datasets",
                                                  os.path.join(GOLDEN, "datasets", "make_golden_nvs_datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIX))


@pytest.fixture(scope="module")
def root(gen, fx, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("nvs_sequences"))
    gen.write_sequences(d, fx)
    return d


@pytest.mark.parametrize("prefetch", [0, 2])
@pytest.mark.parametrize("read", READS)
def test_frames_bit_identical_to_reference(gen, fx, root, cuda_device, read, prefetch):
    dataset, split, kw = gen.READS[read]
    config = gen.REPLICAV2_CONFIG if dataset == "replicav2" else None
    with D.RGBDSequence(dataset, os.path.join(root, dataset), gen.SEQUENCES[dataset], config, device=cuda_device,
                        prefetch=prefetch, split=split, **kw) as seq:
        assert len(seq) == len(fx[read + "_retained"])
        for t in range(len(seq)):
            fr = seq[t]
            assert fr["im"].shape == (3, seq.height, seq.width)
            assert torch.equal(fr["im"].cpu(), torch.from_numpy(fx[read + "_color"][t])), (read, t)
            assert torch.equal(fr["depth"].cpu(), torch.from_numpy(fx[read + "_depth"][t])), (read, t)
            pose = torch.from_numpy(fx[read + "_poses"][t]).to(cuda_device)
            assert torch.equal(fr["gt_w2c"], torch.linalg.inv(pose))
