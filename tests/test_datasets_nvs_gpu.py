"""GPU: the ScanNet++ and ReplicaV2 readers (splatam_b200/datasets.py) through the ingest kernel against the
reference's own dataset classes (tests/golden/datasets/ref_nvs_datasets.npz): colour and depth bit for bit for every
read of both splits -- ScanNet++'s JPEG colour at the exact-2x and a non-2x size, ReplicaV2's PNG colour natively and
downscaled -- with the synchronous and the prefetching reader."""
import pytest
import torch

from dataset_fixtures import sequence, sequence_fixtures

pytestmark = pytest.mark.gpu

READS = ["scannetpp_train", "scannetpp_train_bad", "scannetpp_test", "scannetpp_test_bad", "replicav2_train",
         "replicav2_test", "replicav2_test_sel"]


gen, fx, root = sequence_fixtures("nvs_datasets")


@pytest.mark.parametrize("prefetch", [0, 2])
@pytest.mark.parametrize("read", READS)
def test_frames_bit_identical_to_reference(gen, fx, root, cuda_device, read, prefetch):
    with sequence(gen, root, read, cuda_device, prefetch) as seq:
        assert len(seq) == len(fx[read + "_retained"])
        for t in range(len(seq)):
            fr = seq[t]
            assert fr["im"].shape == (3, seq.height, seq.width)
            assert torch.equal(fr["im"].cpu(), torch.from_numpy(fx[read + "_color"][t])), (read, t)
            assert torch.equal(fr["depth"].cpu(), torch.from_numpy(fx[read + "_depth"][t])), (read, t)
            pose = torch.from_numpy(fx[read + "_poses"][t]).to(cuda_device)
            assert torch.equal(fr["gt_w2c"], torch.linalg.inv(pose))
