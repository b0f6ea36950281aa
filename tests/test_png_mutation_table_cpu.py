"""CPU: the mutation tables of tests/run_png_mutations.py still apply to csrc/png_deflate.cu, png_inflate.cu and image_io.cu
- every anchor occurs exactly once and is changed by its mutation, the GPU test file exists, and only the mutated source
has to be rebuilt for a mutant - so an edit that breaks an anchor is noticed here rather than on the next H100 run."""
import os

from panic3d_b200 import _build
from tests.run_mutations import ROOT, units_including
from tests.run_png_mutations import TARGETS


def test_png_mutation_table_applies_to_the_current_source():
    assert sorted(TARGETS) == ['image_io', 'png_deflate', 'png_inflate']
    for target, (src_name, test_file, mutations) in TARGETS.items():
        assert os.path.isfile(os.path.join(ROOT, test_file)), test_file
        text = open(os.path.join(_build.CSRC, src_name)).read()
        assert len(mutations) >= 4, target
        for name, (old, new) in mutations.items():
            assert old != new, name
            assert text.count(old) == 1, f'{target}: {name}: anchor found {text.count(old)} times in {src_name}'
        assert {os.path.basename(s) for s in units_including(src_name)} == {src_name}, target
