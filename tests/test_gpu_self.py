"""-m gpu: SELF mode (`FastGA A`, SURVEY row a-7) -- the CUDA path against the oracle, which is
pinned against the reference's own self runs in tests/test_oracle_pin.py and tests/test_self_cases.py."""
import numpy as np
import pytest

import oracle_lib as ol
import self_cases as sc
from fastga_b200 import formats, lib
from test_oracle_pin import _self_genomes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["dup", "tandem61", "tandem62", "inverted_dup", "identical_contigs", "palindrome",
                                  "near_diagonal_repeats", "contigs300"] + sorted(sc.GENOMES))
def test_self_mode_bit_exact_vs_oracle(name):
    G = sc.GENOMES[name]() if name in sc.GENOMES else _self_genomes()[name]
    g = formats.genome_from_arrays(G)
    # the device advances a tube across the main diagonal with 0, not the reference's stale bepos; on the
    # divergence genome (only) that keeps sc.DIVERGENT_RECORDS more records
    want = ol.oracle_pipeline_self(g, straddle_zero=(name == "divergence"))
    alns, stats = lib.fastga_self(g)
    assert stats["nseeds"] == want["nseeds"]
    assert stats["nhits"] == want["nhit"]
    assert alns.nraw == want["nraw"]
    assert alns.canonical_lines() == want["lines"]
