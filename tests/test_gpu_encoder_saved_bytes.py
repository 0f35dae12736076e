"""GPU suite: the grad-mode encoder forward (precision 3) returns, byte for byte, what the golden digests record — its
raw outputs and every tensor of its saved-activation buffer (stem, block-0 depthwise and every later ReLU output, the heads'
pre-clamp values) — for SmirkEncoder and each sub-encoder alone at B = 1, 7 and 32.  The fused stem + block-0 kernel
writes the stem and depthwise slots and the block-0 output every later layer reads, so any change to its arithmetic or
its coverage of the tiles shows here."""
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
    m = mg.make_module(name)
    for B in mg.BATCHES:
        assert mg.digests(m, B) == gold["%s/B%d" % (name, B)], "%s at B = %d" % (name, B)
