"""CPU test of how the fused forward kernel reads k_f: the plain fwd3_kernel instantiations (ungated real sequences,
bf16 and fp16) take the channel's k_f block into the unit's shared-memory slot by one bulk copy, so their unit loop
issues no global load (LDG) at all, and wait for the kernel before them (griddepcontrol.wait) before the loop.  The
gated and complex-rows instantiations keep their global loads of k_f (fwd3_r128.cuh, kKfSlot).  Every instantiation stays within the
128-register cap with no local memory.  Reads the SASS of the built library with cuobjdump (skipped where it is not
installed), as test_register_budget.py."""
import re
import subprocess

import pytest

from test_register_budget import _cuobjdump, unit_loop


def _ungated(name):       # template <bool kPlanes, bool kGated, ...>: _Z..fwd3_kernelILb<kPlanes>ELb<kGated>E
    return 'fwd3_kernelILb0ELb0E' in name


@pytest.fixture(scope='module')
def fwd3():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not available')
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    sass = subprocess.run([tool, '-sass', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    res = subprocess.run([tool, '-res-usage', _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', sass)[1:]:
        name = chunk.split('\n', 1)[0].strip()
        if 'fwd3_kernel' in name:
            funcs[name] = {'ins': [(int(a, 16), t) for a, t in re.findall(r'/\*([0-9a-f]{4,})\*/\s+([^;]*);', chunk)]}
    for name, rest in re.findall(r'Function (\S+):\s*\n?\s*(REG:\d+[^\n]*)', res):
        if name in funcs:
            funcs[name]['reg'] = int(re.search(r'REG:(\d+)', rest).group(1))
            funcs[name]['local'] = int(re.search(r'LOCAL:(\d+)', rest).group(1))
    return funcs


def test_every_instantiation_found(fwd3):
    assert len(fwd3) == 8 and sum(_ungated(n) for n in fwd3) == 2, sorted(fwd3)


def test_no_global_load_in_ungated_unit_loop(fwd3):
    bad = {}
    for name, f in fwd3.items():
        if not _ungated(name):
            continue
        head, back = unit_loop(f['ins'])
        ldg = [f'{a:#x}: {t.strip()}' for a, t in f['ins'] if head <= a <= back and re.search(r'\bLDG\b', t)]
        if ldg:
            bad[name] = (len(ldg), ldg[:4])
    assert not bad, f'global loads inside the unit loop: {bad}'


def test_ungated_waits_for_the_kernel_before(fwd3):
    # griddepcontrol.wait (ACQBULK) before the unit loop: the grid is launched as a programmatic dependent
    for name, f in fwd3.items():
        if _ungated(name):
            head, _ = unit_loop(f['ins'])
            assert any(a < head and re.search(r'\bACQBULK\b', t) for a, t in f['ins']), name


def test_registers_and_local_memory(fwd3):
    for name, f in fwd3.items():
        assert 'reg' in f, f'no resource usage for {name}'
        assert f['reg'] <= 128, (name, f['reg'])
        assert f['local'] == 0, (name, f['local'])
