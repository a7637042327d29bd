"""-m gpu: SELF mode (`FastGA A`, SURVEY row a-7) -- the CUDA path against the oracle, which is
pinned against the reference's own self runs in tests/test_oracle_pin.py."""
import numpy as np
import pytest

import oracle_lib as ol
from fastga_b200 import formats, lib
from test_oracle_pin import _self_genomes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["dup", "tandem61", "tandem62", "contigs300"])
def test_self_mode_bit_exact_vs_oracle(name):
    g = formats.genome_from_arrays(_self_genomes()[name])
    want = ol.oracle_pipeline_self(g)
    alns, stats = lib.fastga_self(g)
    assert stats["nseeds"] == want["nseeds"]
    assert stats["nhits"] == want["nhit"]
    assert alns.nraw == want["nraw"]
    assert alns.canonical_lines() == want["lines"]
