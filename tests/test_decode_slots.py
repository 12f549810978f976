"""CPU tests of decoding with one position per batch row (bffc_conv_state_fill_slots / bffc_conv_step_slots,
HyenaDecoder / LongConvDecoder with slots=True).

1. Every BFFC_ERR_INVALID rule of the three entry points, with fake pointers, before the device is looked at: the
   rules the shared calls apply, and n, L, null or misaligned slots / lengths / pos.
2. The slot workspace formula, mirrored in Python; the shared formula is unchanged.
3. The launch grids of the slot calls for B, H up to 131073 / 65600, with the mirror of test_decode.py.
4. The Python state and position layout against the library's sizes.
5. The host validation of lengths and slots: duplicates, out of range, n > B, L > max_len.
"""
import ctypes

import pytest
import torch

from test_decode import BFFC_ERR_INVALID, BAD_COMMON, CHUNK, GOOD, GRID_YZ, INT_MAX, MAX_T, THREADS, fill_grid, \
    step_grids

P = ctypes.c_void_p


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import _lib
    return _lib


def _state_bytes(lib, a):
    return lib.lib().bffc_conv_state_bytes(a['B'], a['H'], a['max_len'], a['K'], a['residual'], 0) or 1 << 30


def _fill_slots(lib, **kw):
    a = dict(GOOD, n=2, u=P(1 << 20), pre=P(2 << 20), post=P(3 << 20), w=P(4 << 20), bias=P(4 << 20),
             state=P(5 << 20), pos=P(6 << 20), slots=P(11 << 20), lengths=P(12 << 20), bs=None, state_bytes=None)
    a.update(kw)
    bs = a['H'] * a['L'] if a['bs'] is None else a['bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    rc = lib.lib().bffc_conv_state_fill_slots(a['u'], bs, a['pre'], bs, a['post'], bs, a['w'], a['bias'], a['w'],
                                              a['bias'], a['w'], a['bias'], a['w_dtype'], a['K'], a['padding'],
                                              a['dtype'], a['B'], a['H'], a['n'], a['L'], a['slots'], a['lengths'],
                                              a['max_len'], a['residual'], a['state'], sb, a['pos'], P(0))
    return rc, lib.lib().bffc_last_error().decode()


def _step_slots(lib, **kw):
    a = dict(GOOD, u=P(1 << 20), pre=P(2 << 20), post=P(3 << 20), w=P(4 << 20), bias=P(4 << 20), state=P(5 << 20),
             pos=P(6 << 20), k=P(7 << 20), k2=P(8 << 20), y=P(9 << 20), ws=P(10 << 20), bs=None, y_bs=None,
             state_bytes=None, ws_bytes=1 << 30)
    a.update(kw)
    bs = a['H'] * a['T'] if a['bs'] is None else a['bs']
    y_bs = a['H'] * a['T'] if a['y_bs'] is None else a['y_bs']
    sb = _state_bytes(lib, a) if a['state_bytes'] is None else a['state_bytes']
    rc = lib.lib().bffc_conv_step_slots(a['u'], bs, a['pre'], bs, a['post'], bs, a['k'], a['Lk'], a['k2'], a['Lk2'],
                                        a['w'], a['bias'], a['w'], a['bias'], a['w'], a['bias'], a['w_dtype'],
                                        a['K'], a['padding'], a['dtype'], a['state'], sb, a['pos'], a['y'], y_bs,
                                        a['B'], a['H'], a['T'], a['max_len'], a['ws'], a['ws_bytes'], P(0))
    return rc, lib.lib().bffc_last_error().decode()


# ----------------------------------------------------------------------------------------------- argument checks
@pytest.mark.parametrize('bad,msg', BAD_COMMON)
@pytest.mark.parametrize('fn', ['state_fill_slots', 'step_slots'])
def test_invalid_arguments(lib, fn, bad, msg):
    rc, err = (_fill_slots if fn == 'state_fill_slots' else _step_slots)(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err and f'bffc_conv_{fn}' in err, err


@pytest.mark.parametrize('bad,msg', [
    (dict(L=-1), 'shape'), (dict(L=101), 'shape'),
    (dict(n=3), 'n=3'), (dict(n=0), 'n=0'), (dict(n=-1), 'n=-1'),
    (dict(slots=P(0)), 'slots / lengths'), (dict(lengths=P(0)), 'slots / lengths'),
    (dict(slots=P((11 << 20) + 2)), 'slots / lengths'), (dict(lengths=P((12 << 20) + 1)), 'slots / lengths'),
    (dict(pos=P(0)), 'pos'), (dict(pos=P((6 << 20) + 4)), 'pos')])
def test_invalid_fill_slots_arguments(lib, bad, msg):
    rc, err = _fill_slots(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


@pytest.mark.parametrize('bad,msg', [
    (dict(T=0), 'T='), (dict(T=65), 'T='), (dict(T=101, max_len=100), 'T='),
    (dict(k=P(0)), 'k null'), (dict(Lk=0), 'Lk='), (dict(Lk=101), 'Lk='), (dict(Lk2=101), 'Lk2='),
    (dict(y=P(0)), 'y null'), (dict(y_bs=3), 'batch stride'),
    (dict(ws=P(0)), 'workspace'), (dict(ws=P((10 << 20) + 8)), 'workspace'), (dict(pos=P(0)), 'pos')])
def test_invalid_step_slots_arguments(lib, bad, msg):
    rc, err = _step_slots(lib, **bad)
    assert rc == BFFC_ERR_INVALID and msg in err, err


def test_step_slots_needs_the_slot_workspace(lib):
    """the shared workspace size is one header short of the snapshot of B > 32 positions"""
    B, H, T, Lk, Lk2 = 100, 4, 1, 100, 50
    shared = lib.lib().bffc_conv_step_workspace_bytes(B, H, T, Lk, Lk2)
    slots = lib.lib().bffc_conv_step_slots_workspace_bytes(B, H, T, Lk, Lk2)
    assert slots > shared
    rc, err = _step_slots(lib, B=B, ws_bytes=shared)
    assert rc == BFFC_ERR_INVALID and f'{slots} bytes' in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks that valid arguments reach the device check')
@pytest.mark.parametrize('fn', ['fill_slots', 'step_slots'])
@pytest.mark.parametrize('kw', [{}, dict(K=1, padding=0), dict(K=32, padding=31, w_dtype=0), dict(T=64),
                                dict(pre=P(0), post=P(0), w=P(0), bias=P(0), residual=0, k2=P(0)), dict(L=0),
                                dict(n=1), dict(B=1, n=1)])
def test_valid_arguments_reach_the_device_check(lib, fn, kw):
    rc, err = (_fill_slots if fn == 'fill_slots' else _step_slots)(lib, **kw)
    assert rc == 3 and 'no CUDA device' in err, err


# ----------------------------------------------------------------------------------------------- workspace
def slot_workspace_bytes(B, H, T, Lk, Lk2):
    """decode_step.cuh: a header of B int64 positions (2B floats rounded up to 64), s_postgate, the partials"""
    header = -(-2 * B // 64) * 64
    return 4 * (header + B * H * T * (1 + -(-Lk // CHUNK) + -(-Lk2 // CHUNK)))


@pytest.mark.parametrize('B', [1, 2, 31, 32, 33, 64, 65, 1000, 65537])
@pytest.mark.parametrize('H,T,Lk,Lk2', [(1, 1, 1, 0), (4, 3, 5000, 0), (4, 64, 5000, 2049), (768, 1, 8192, 4096)])
def test_slot_workspace_bytes(lib, B, H, T, Lk, Lk2):
    l = lib.lib()
    assert l.bffc_conv_step_slots_workspace_bytes(B, H, T, Lk, Lk2) == slot_workspace_bytes(B, H, T, Lk, Lk2)
    if B <= 32:                            # the shared header (64 floats) holds 32 positions
        assert l.bffc_conv_step_slots_workspace_bytes(B, H, T, Lk, Lk2) == \
            l.bffc_conv_step_workspace_bytes(B, H, T, Lk, Lk2)


def test_slot_workspace_bytes_refusals(lib):
    l = lib.lib()
    for args in [(0, 1, 1, 1, 0), (1, 0, 1, 1, 0), (1, 1, 0, 1, 0), (1, 1, 65, 1, 0), (1, 1, 1, 0, 0), (1, 1, 1, 1, -1)]:
        assert l.bffc_conv_step_slots_workspace_bytes(*args) == 0, args
    # the shared formula is what it was: a 64-float header whatever B is
    assert l.bffc_conv_step_workspace_bytes(100, 4, 3, 5000, 0) == 4 * (64 + 100 * 12 * (1 + 3))


# ----------------------------------------------------------------------------------------------- launch grids
def fill_slots_grid(n, H, L):
    return (-(-max(L, 1) // THREADS), min(H, GRID_YZ), min(n, GRID_YZ))


EXT = [1, 65535, 65536, 65537, 65600, 131073]


@pytest.mark.parametrize('B', EXT)
@pytest.mark.parametrize('H', EXT)
def test_grids_within_limits(B, H):
    for max_len in (64, 8192, 1 << 20):
        for T in (1, MAX_T):
            g1, g2 = step_grids(B, H, T, max_len, max_len)         # the slot step launches the shared step's grids
            for n in {1, B}:
                g = fill_slots_grid(n, H, max_len)
                assert 1 <= g[0] <= INT_MAX and 1 <= g[1] <= GRID_YZ and 1 <= g[2] <= GRID_YZ, g
                assert -(-n // g[2]) * g[2] >= n                   # every prompt row is reached over gridDim.z
            assert fill_slots_grid(B, H, max_len) == fill_grid(B, H, max_len)
            # the slot loops over the B columns keep their int index below 2^31 through the last increment: the
            # reach and snapshot loop of step_lags (b += kThreads) and the position advance of step_finish
            # (c += gridDim.x * kThreads)
            assert B - 1 + THREADS <= INT_MAX and B - 1 + g2[0] * THREADS <= INT_MAX
            # a snapshot column b is written by the chunk-0 block with blockIdx.y = b % gridDim.y: exactly one block
            assert all(sum(1 for y in range(g1[1]) if b % g1[1] == y) == 1 for b in {0, B // 2, B - 1})
            # the header of B int64 positions and the column indices stay in int
            assert 2 * B <= INT_MAX and -(-2 * B // 64) * 64 <= INT_MAX


# ----------------------------------------------------------------------------------------------- Python layout
@pytest.mark.parametrize('B,H,n,K,res', [(1, 1, 1, 1, 0), (5, 8, 256, 4, 1), (65537, 1, 256, 3, 0)])
def test_python_state_and_position_layout(lib, B, H, n, K, res):
    """a slot decoder's state is the shared decoder's state (decode.state_layout against the library); the position
    array the decoders allocate (decode.position_array) is the include/bffc.h layout; the slot workspace query is the
    slot formula"""
    from flashfftconv.decode import position_array, state_layout
    zc, vc, total = state_layout(B, H, n, K, res)
    assert total == lib.lib().bffc_conv_state_bytes(B, H, n, K, res, 0)
    pos = position_array(B, True, 'cpu')
    assert pos.dtype == torch.int64 and pos.shape == (2, B) and pos.is_contiguous()
    base = pos.data_ptr()
    for b in {0, B // 2, B - 1}:                   # pos[0][b] at pos + b, pos[1][b] at pos + B + b
        assert pos[0, b].data_ptr() == base + 8 * b and pos[1, b].data_ptr() == base + 8 * (B + b)
    assert (pos[0] == -1).all() and (pos[1] == 0).all()            # every slot idle, no status
    shared = position_array(B, False, 'cpu')                        # the int64[2] of the shared calls: (2, 1) as 2
    assert shared.dtype == torch.int64 and shared.shape == (2,) and shared.tolist() == [0, 0]
    assert lib.lib().bffc_conv_step_slots_workspace_bytes(B, H, 1, n, 0) == slot_workspace_bytes(B, H, 1, n, 0)


# ----------------------------------------------------------------------------------------------- host validation
def _host_decoder(slots=True, batch=4, max_len=100):
    """a decoder without device state: enough for the host-side validation of an admission"""
    from flashfftconv.decode import HyenaDecoder
    d = object.__new__(HyenaDecoder)
    d.slots, d.batch, d.max_len = slots, batch, max_len
    return d


@pytest.mark.parametrize('n,L,lengths,slots,msg', [
    (2, 10, [3, 4], [1, 1], 'not distinct'),
    (2, 10, [3, 4], [0, 4], 'outside'), (2, 10, [3, 4], [-1, 0], 'outside'),
    (2, 10, [3, 11], [0, 1], 'lengths'), (2, 10, [-1, 3], [0, 1], 'lengths'),
    (2, 10, [3], [0, 1], '1 lengths for 2 prompts'), (2, 10, [3, 4], [0], '1 slots for 2 prompts'),
    (5, 10, [1] * 5, None, '5 prompts for 4 slots'),
    (3, 10, [1] * 3, None, 'every one of the 4 slots'),
    (1, 101, [5], [0], 'exceeds max_len'),
    (1, 10, None, [0], 'lengths=')])
def test_admission_is_validated_on_the_host(n, L, lengths, slots, msg):
    d = _host_decoder()
    with pytest.raises(ValueError, match=msg):
        d._admission(n, L, lengths, slots)


def test_admission_accepts_host_sequences_and_cpu_tensors():
    d = _host_decoder()
    assert d._admission(4, 10, [0, 1, 10, 5], None) == ([0, 1, 2, 3], [0, 1, 10, 5])
    assert d._admission(2, 10, torch.tensor([3, 7]), torch.tensor([3, 0], dtype=torch.int32)) == ([3, 0], [3, 7])
    assert d._admission(1, 0, (0,), (2,)) == ([2], [0])
    with pytest.raises(ValueError, match='CPU integer tensor'):
        d._admission(2, 10, torch.tensor([3.0, 7.0]), None)


def test_slot_release_validates_slots():
    d = _host_decoder()
    for bad, msg in [([4], 'outside'), ([0, 0], 'not distinct'), (None, 'reset')]:
        with pytest.raises(ValueError, match=msg):
            d.release(bad)


def test_position_book_mirror():
    """the host mirror follows admissions, steps (active slots only) and ragged extends, refuses what would pass max_len
    or extend an idle slot, and is forgotten under capture (the device then decides)"""
    from flashfftconv.decode_state import PositionBook
    b = PositionBook(3, True, 'cpu', 100)
    b._put([0, 2], [10, 5])
    assert b._host_pos == [10, -1, 5]
    b._advance(4, False)
    assert b._host_pos == [14, -1, 9]
    b._advance(8, False, ([2, 0], [3, 8]))
    assert b._host_pos == [22, -1, 12]
    with pytest.raises(ValueError, match=r'slots \[1\] are idle'):
        b._check_room(4, False, ([1], [4]))
    with pytest.raises(ValueError, match=r'slots \[0\] at positions \[22\] \+ \[79\] tokens exceed'):
        b._check_room(79, False, ([0, 2], [79, 1]))
    with pytest.raises(ValueError, match=r'slots \[0\] at positions \[22\] \+ 79 tokens exceed'):
        b._check_room(79, False)
    b._check_room(78, False)
    far = PositionBook(3, True, 'cpu')
    far._follow(b, None, False)
    assert far._host_pos == [22, -1, 12]
    b._advance(1, False, ([2], [1]))
    far._follow(b, [2], False)
    assert far._host_pos == [22, -1, 13]
    b._advance(1, True)
    assert b._host_pos is None
    b._check_room(1000, False)
    far._follow(b, None, False)
    assert far._host_pos is None
    b._restart()
    assert b._host_pos == [-1] * 3 and b._pos.tolist() == [[-1] * 3, [0] * 3]
    s = PositionBook(1, False, 'cpu', 10)
    s._put(None, 6)
    s._advance(3, False, None)
    assert s._host_pos == 9
    with pytest.raises(ValueError, match='exceeds max_len'):
        s._check_room(2, False)
    assert s._admission(1, 10, None, None) == (None, None)
    with pytest.raises(ValueError, match='exceeds max_len'):
        s._admission(1, 11, None, None)


def test_shared_decoder_refuses_slot_calls():
    d = _host_decoder(slots=False)
    with pytest.raises(RuntimeError, match='slots=True'):
        d.release([0])
    with pytest.raises(RuntimeError, match='slots=True'):
        d.positions
    s = _host_decoder(slots=True)
    with pytest.raises(RuntimeError, match='positions'):
        s.pos
