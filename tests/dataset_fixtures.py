"""The tiny on-disk sequences of the dataset golden generators (tests/golden/datasets/make_golden_datasets.py and
make_golden_nvs_datasets.py) and the readers over them, shared by the dataset, NVS and SplaTAM-S tests.

A test module takes the fixtures with `gen, fx, root = sequence_fixtures("datasets")` (or "nvs_datasets"); they are
module-scoped, so each module writes its own sequence directory once."""
import os

import numpy as np
import pytest

from util import GOLDEN, load
from splatam_b200 import datasets as D


def sequence_fixtures(name):
    """Fixtures `gen` (the generator make_golden_<name>.py), `fx` (the arrays of ref_<name>.npz) and `root` (a
    directory with the generator's sequences written from those arrays)."""
    arrays = os.path.join(GOLDEN, "datasets", "ref_%s.npz" % name)

    @pytest.fixture(scope="module")
    def gen():
        return load(os.path.join(GOLDEN, "datasets", "make_golden_%s.py" % name))

    @pytest.fixture(scope="module")
    def fx():
        return dict(np.load(arrays))

    @pytest.fixture(scope="module")
    def root(gen, tmp_path_factory):
        d = str(tmp_path_factory.mktemp(name))
        gen.write_sequences(d, dict(np.load(arrays)))
        return d

    return gen, fx, root


def _read(gen, root, read):
    """Positional and keyword arguments of SequenceFiles / RGBDSequence for one entry of the generator's READS:
    (dataset, kw) in make_golden_datasets, (dataset, split, kw) in make_golden_nvs_datasets."""
    dataset, *split, kw = gen.READS[read]
    if split:
        config, kw = (gen.REPLICAV2_CONFIG if dataset == "replicav2" else None), dict(kw, split=split[0])
    else:
        config = gen.config(dataset)
    return (dataset, os.path.join(root, dataset), gen.SEQUENCES[dataset], config), kw


def files_of(gen, root, read):
    args, kw = _read(gen, root, read)
    return D.SequenceFiles(*args, **kw)


def sequence(gen, root, read, device, prefetch, **extra):
    args, kw = _read(gen, root, read)
    return D.RGBDSequence(*args, device=device, prefetch=prefetch, **dict(kw, **extra))
