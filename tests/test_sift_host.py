"""CPU: the SIFT extraction surface of the C++ host -- SiftExtractionOptions with the C++ defaults
(R:pipeline/extract_features.h:78-139), pycolmap's three overrides on Sift() (R:pycolmap/feature/sift.h:99-102), dict /
keyword construction, pickle, the Normalization string constructor, the argument checks that come before any GPU work,
and no CPU fallback."""
import pickle

import numpy as np
import pytest

from helpers.native_import import load_native

nat = load_native()


def test_defaults():
    o = nat.SiftExtractionOptions().todict()
    assert o == dict(num_threads=-1, gpu_index="-1", max_image_size=3200, max_num_features=8192, first_octave=-1,
                     num_octaves=4, octave_resolution=3, peak_threshold=0.02 / 3, edge_threshold=10.0,
                     estimate_affine_shape=False, max_num_orientations=2, upright=False, darkness_adaptivity=False,
                     domain_size_pooling=False, dsp_min_scale=1.0 / 6, dsp_max_scale=3.0, dsp_num_scales=10,
                     normalization=nat.Normalization.L1_ROOT)
    s = nat.Sift().options
    assert (s.peak_threshold, s.first_octave, s.max_image_size) == (0.01, 0, 7000)
    assert s.max_num_features == 8192 and s.octave_resolution == 3 and s.edge_threshold == 10.0
    assert nat.Sift().device == nat.Device.cuda


def test_construction_pickle_and_enum():
    o = nat.SiftExtractionOptions({"peak_threshold": 0.02, "normalization": "L2", "upright": True})
    assert o.peak_threshold == 0.02 and o.normalization == nat.Normalization.L2 and o.upright
    k = nat.SiftExtractionOptions(max_num_features=100)
    assert k.max_num_features == 100 and k.first_octave == -1
    assert pickle.loads(pickle.dumps(o)).todict() == o.todict()
    assert nat.Normalization("L1_ROOT") == nat.Normalization.L1_ROOT
    with pytest.raises(IndexError):
        nat.Normalization("L3")
    with pytest.raises(AttributeError):
        nat.SiftExtractionOptions({"no_such_field": 1})
    s = nat.Sift({"max_num_orientations": 3})
    assert s.options.max_num_orientations == 3 and s.options.peak_threshold == 0.02 / 3


@pytest.mark.parametrize("bad", [dict(max_image_size=0), dict(max_num_features=0), dict(octave_resolution=0),
                                 dict(peak_threshold=0.0), dict(edge_threshold=-1.0), dict(max_num_orientations=0),
                                 dict(num_octaves=0), dict(estimate_affine_shape=True), dict(domain_size_pooling=True),
                                 dict(darkness_adaptivity=True), dict(gpu_index="0,1")])
def test_option_checks(bad):
    with pytest.raises(ValueError, match="Check Failed"):
        nat.Sift(nat.SiftExtractionOptions(bad))


def test_image_checks():
    s = nat.Sift({"max_image_size": 64})
    with pytest.raises(TypeError):
        s.extract(np.zeros((16, 16)))                       # float64
    with pytest.raises(TypeError):
        s.extract(np.zeros((16, 16), np.int32))
    for img in [np.zeros((4, 4, 3), np.uint8), np.zeros((0, 16), np.uint8), np.zeros((65, 16), np.uint8),
                np.zeros((16, 65), np.uint8), np.full((16, 16), 1.5, np.float32), np.full((16, 16), np.nan, np.float32),
                np.full((16, 16), -0.1, np.float32)]:
        with pytest.raises(ValueError, match="Check Failed"):
            s.extract(img)
    with pytest.raises(ValueError, match="Check Failed"):
        s.extract_batch([np.zeros((16, 16), np.uint8), np.zeros((65, 16), np.uint8)])
    with pytest.raises(ValueError):
        nat.Sift(device=nat.Device.cpu)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    with pytest.raises(Exception, match="device|CUDA|sm_90"):
        nat.Sift().extract(np.zeros((32, 32), np.uint8))
