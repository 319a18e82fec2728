"""The VGG16 feature-reconstruction loss gives the bits of the build it was frozen from (tests/golden/vgg_bits.npz): values
and d value / d rec for every option set of tests/_vgg_oracle.OPTION_SETS."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_vgg_term_is_unchanged_bit_for_bit():
    from tests import _vgg_oracle as OV
    from tests.golden.make_vgg_bits_golden import vgg_bits
    z = np.load(os.path.join(GOLDEN, 'vgg_bits.npz'))
    got = vgg_bits()
    assert len(got) == 2 * len(OV.OPTION_SETS) == len(z.files)
    for k, v in got.items():
        assert np.array_equal(v.view(np.uint32), z[k].view(np.uint32)), k
