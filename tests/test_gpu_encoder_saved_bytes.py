"""GPU suite: the grad-mode encoder forward returns, byte for byte, what the golden digests record — its
raw outputs and every tensor of its saved-activation buffer (stem, block-0 depthwise and every later ReLU output, the heads'
pre-clamp values) — for SmirkEncoder and each sub-encoder alone at B = 1, 7 and 32, at precisions 0 to 3.  The stem
kernels write the stem and depthwise slots and the block-0 output every later layer reads, so any change to their arithmetic
or their coverage of the map shows here."""
import json

import pytest

import make_golden_encoder_saved as mg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    with open(mg.GOLD) as fh:
        return json.load(fh)


@pytest.mark.parametrize("name", mg.MODULES)
def test_forward_saved_bytes_match_golden(native_lib, gold, name):
    for p in mg.PRECISIONS:
        m = mg.make_module(name, p)
        for B in mg.BATCHES:
            assert mg.digests(m, B) == gold[mg.key(p, name, B)], "%s at precision %d, B = %d" % (name, p, B)
