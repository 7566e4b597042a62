"""CPU tests (no GPU) of tecogan_b200.VGGFeatureExtractor: which feature indices it accepts, its state_dict against
the reference's VGGFeatureExtractor (built with the same seeded VGG19 stub), the shapes of the features it returns,
and its argument checks."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                            # noqa: E402
import refimport                                    # noqa: E402

RELUS = (1, 3, 6, 8, 11, 13, 15, 17, 20, 22, 24, 26, 29, 31, 33, 35)


@pytest.fixture(scope='module', autouse=True)
def seeded_vgg19():
    refimport.stub_pretrained_vgg19()      # no download: seeded weights of the same architecture


def _reference_class():
    if not refimport.available():
        pytest.skip('reference not installed (oracle/_ref)')
    refimport._prepare()
    from models.networks.vgg_nets import VGGFeatureExtractor
    return VGGFeatureExtractor


@pytest.mark.parametrize('idx', [(8, 17, 26, 35), RELUS, (35,), (1,), (26, 8), (3, 22, 33)])
def test_every_relu_index_is_accepted(idx):
    vgg = T.VGGFeatureExtractor(idx)
    assert vgg.feature_indexs == sorted(idx)


@pytest.mark.parametrize('idx', [(0,), (2,), (4,), (9,), (36,), (37,), (-1,), (8, 7), (8, 17, 26, 34), (8.0,)])
def test_other_indices_raise(idx):
    with pytest.raises(ValueError):
        T.VGGFeatureExtractor(idx)


def test_state_dict_keys_and_values_equal_the_reference():
    Ref = _reference_class()
    ref, ours = Ref(), T.VGGFeatureExtractor()
    rs, os_ = ref.state_dict(), ours.state_dict()
    assert list(rs) == list(os_)
    for k in rs:
        assert torch.equal(rs[k], os_[k]), k
    assert all(not p.requires_grad for p in ours.parameters())
    ours.load_state_dict(ref.state_dict())           # what check_reference_gan_training_integration does


@pytest.mark.parametrize('idx', [(8, 17, 26, 35), RELUS, (3, 22)])
@pytest.mark.parametrize('h,w', [(64, 64), (70, 90), (17, 23), (16, 16), (33, 48)])
def test_feature_shapes_match_the_reference(idx, h, w):
    ref = _reference_class()(idx)
    # the reference's forward runs every layer, so below 32 pixels its last pool fails: run its layers up to the
    # deepest requested index, which is all the features it returns depend on
    out, want = (torch.rand(2, 3, h, w) - ref.mean) / ref.std, []
    with torch.no_grad():
        for i in range(max(idx) + 1):
            out = ref.features[i](out)
            if i in ref.feature_indexs:
                want.append(tuple(out.shape))
    assert T.VGGFeatureExtractor(idx).feature_shapes(2, h, w) == want


def test_misuse_raises():
    vgg = T.VGGFeatureExtractor()
    with pytest.raises(T.TecoganB200Error):
        vgg(torch.rand(1, 3, 32, 32))                # CPU tensor: no CPU fallback
