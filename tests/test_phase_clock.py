"""CPU test of the fused forward kernel's phase clock (-DBFFC_PHASE_CLOCK, fwd3_r128.cuh, tools/fwd_phases.py): it is a
diagnostic build only, so the normal build's fwd3_kernel instantiations read no clock and the library exports no
phase-clock entry point.  Reads the SASS of the built library with cuobjdump (skipped where it is not installed), as
test_register_budget.py."""
import ctypes
import re
import subprocess

import pytest

from test_register_budget import _cuobjdump


def test_normal_build_has_no_phase_clock():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    sass = subprocess.run([tool, '-sass', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    found = 0
    for chunk in re.split(r'\n\s*Function : ', sass)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if 'fwd3_kernel' in name:
            found += 1
            assert not re.search(r'SR_CLOCK', chunk), name
    assert found == 8
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert not hasattr(lib, 'bffc_phase_clock')
