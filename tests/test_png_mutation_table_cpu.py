"""CPU: the mutation table of tests/run_png_mutations.py still applies to csrc/png_deflate.cu - every anchor occurs exactly
once and is changed by its mutation, the GPU test file exists, and only png_deflate.cu has to be rebuilt for a mutant - so an
edit that breaks an anchor is noticed here rather than on the next H100 run."""
import os

from panic3d_b200 import _build
from tests.run_mutations import ROOT, units_including
from tests.run_png_mutations import TARGET


def test_png_mutation_table_applies_to_the_current_source():
    src_name, test_file, mutations = TARGET
    assert os.path.isfile(os.path.join(ROOT, test_file)), test_file
    text = open(os.path.join(_build.CSRC, src_name)).read()
    assert len(mutations) >= 6
    for name, (old, new) in mutations.items():
        assert old != new, name
        assert text.count(old) == 1, f'{name}: anchor found {text.count(old)} times in {src_name}'
    assert {os.path.basename(s) for s in units_including(src_name)} == {src_name}
