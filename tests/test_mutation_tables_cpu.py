"""CPU: the mutation tables of tests/run_mutations.py still apply to the current sources - every anchor occurs exactly once
in its kernel file or header and is changed by its mutation, every target's GPU test file exists, and a header target's
mutants rebuild the units that include it - so an edit that breaks an anchor is noticed here rather than on the next H100
run."""
import os

import pytest

from panic3d_b200 import _build
from tests.run_mutations import ROOT, TARGETS, units_including


@pytest.mark.parametrize('target', sorted(TARGETS))
def test_mutation_table_applies_to_the_current_source(target):
    src_name, test_file, mutations = TARGETS[target]
    assert os.path.isfile(os.path.join(ROOT, test_file)), test_file
    text = open(os.path.join(_build.CSRC, src_name)).read()
    for name, (old, new) in mutations.items():
        assert old != new, name
        assert text.count(old) == 1, f'{name}: anchor found {text.count(old)} times in {src_name}'
    units = {os.path.basename(s) for s in units_including(src_name)}
    if src_name.endswith('.cu'):
        assert units == {src_name}
    else:
        assert units >= {'render_v1.cu', 'render_backward.cu'}, units
