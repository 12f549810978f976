"""CPU mirror of every launch grid that depends on the batch B or the channel count H (no GPU needed).

CUDA refuses a launch whose gridDim.x exceeds 2^31 - 1 or whose gridDim.y / gridDim.z exceeds 65535; the library turns
that into BFFC_ERR_CUDA ("invalid configuration argument").  Several launches put channels, batch pairs or channel pairs
in gridDim.y / z, so every one of them walks those in groups of at most kMaxGridYZ = 65535 (bffc.cu):

1. chunk_view caps a composite-size chunk at 65535 channels and 65535 batch pairs.  The CUDA-core level-0 stage launches
   (.., channels, pairs) for the chunk; at seqlen 16384 the 4 GiB plane budget alone allows 65536 (pair, channel) items
   per forward chunk, one past the limit for H >= 65536 with B <= 2, or B >= 131071.
2. bffc_kf_pack(_rfft) and bffc_dkf_unpack(_half) put H in gridDim.y or z: they launch once per 65535 channels.
3. The composite filter-side transforms size their channel group from the caller's workspace; a group is at most 65534
   channels (the row launch puts channels in gridDim.y, and a group is a whole number of channel pairs).

The mirror below restates those grids in Python for every seqlen, forward and backward, gated and ungated, for B and H
in {1, 65535, 65536, 65537, 131070 .. 131073, 2^20}, and asserts the limits for every launch.  The short-filter level-0
kernels (bffc_fwd_short_strided, bffc_bwd_short_strided) launch the same grid as the plain ones, so their entries restate
it rather than check anything of their own; tests/test_extents_gpu.py runs them on the device past the cap.
`rules='parent'` restates the grids as they were before these caps; test_parent_rules_fail_at_items_1_to_3 checks that the sweep then fails, and fails exactly at items 1-3 above: the 16K forward level-0 stage (the plain and the
short-filter kernels) at H >= 65536 with B <= 2 or at B >= 131071, every pack / unpack at H >= 65536, and the
filter-side launches of a workspace of more than 32767 channel pairs.  Nothing else fails.

Persistent launches (the fused kernel, the dk_f kernel, the tensor-core outer stage) run at most one block per SM, so
their grid is never the problem; their unit counts are `int` fields, checked here for every shape whose 16-bit
(B, H, L) tensor fits an 80 GB device.
"""
import itertools

import pytest

from test_chunked_gpu import GRID_YZ, _chunk_view, _nlev

K, M = 1024, 1024 * 1024
SIZES = [256, 512, 1024, 2048, 4096, 8192, 16 * K, 32 * K, 64 * K, 128 * K, 256 * K, 512 * K, M, 2 * M, 4 * M]
EXTENTS = [1, 65535, 65536, 65537, 131070, 131071, 131072, 131073, 1 << 20]
GRID_X = (1 << 31) - 1
INT_MAX = (1 << 31) - 1
NUM_SMS = 132                  # H100 SXM; persistent grids are min(units, SMs) blocks
DEVICE_BYTES = 80 * 10 ** 9
OUTER = {16 * K: (2, 1), 32 * K: (4, 1), 64 * K: (8, 1), 128 * K: (8, 2), 256 * K: (8, 4), 512 * K: (8, 8),
         M: (128, 1), 2 * M: (128, 2), 4 * M: (128, 4)}


def _ne(N):
    return max(N, 8192)


def _groups(n, size):
    """distinct group sizes of n items walked in groups of `size`: the full group and the ragged last one"""
    return sorted({min(size, n)} | ({n % size} if n % size else set()))


# ----------------------------------------------------------------------------- the grids
def _chunk_shapes(N, B, H, sets, rules):
    """(chunks, distinct (members, channels) chunk shapes) of for_each_chunk"""
    cb, ch = _chunk_view(N, B, H, sets, cap=None if rules == 'parent' else GRID_YZ)
    n = -(-B // cb) * -(-H // ch)
    return n, [(b, h) for b in _groups(B, cb) for h in _groups(H, ch)]


def _conv_launches(N, B, H, gated, backward, rules):
    """(launch name, grid, persistent units) of one bffc_fwd_strided / bffc_bwd_strided call, and with the short filter
    (bffc_fwd_short_strided / bffc_bwd_short_strided: the level-0 kernels of the same grids).  Chunked launches are listed
    once per distinct chunk shape."""
    out = []
    if N <= 8192:                                   # fused kernel, dk_f kernel on tiles: persistent
        per_unit = 2 * (8192 // N) if N < 8192 else 2
        units = H * -(-B // per_unit)
        passes = (2 if gated else 1) if backward else 1
        out += [('fused', (min(-(-units // 2), NUM_SMS), 1, 1), units)] * passes
        if backward:
            out.append(('dkf tiles', (min(units, NUM_SMS), 1, 1), units))
        return out
    R0, R1 = OUTER[N]
    nlev = _nlev(N)
    _, shapes = _chunk_shapes(N, B, H, nlev + (1 if backward else 0), rules)
    for b, h in shapes:
        pairs = (b + 1) // 2
        if R0 == 128:                               # tensor-core level 0: persistent
            units = pairs * h * (N // 128 // 64)
            out.append(('tc level 0', (min(-(-units // 2), NUM_SMS), 1, 1), units))
        else:
            cb = (N // R0) // (8 * 128)
            for name in ('cc level 0', 'cc level 0 short'):
                out.append((name, (cb, h, pairs), None))
        if R1 > 1:
            out.append(('cc level 1', (pairs * h * R0, (N // (R0 * R1)) // (8 * 128), 1), None))
        units = pairs * h * (N // 8192)
        out.append(('fused planes', (min(-(-units // 2), NUM_SMS), 1, 1), units))
        if backward:
            out.append(('dkf planes', (min(units, NUM_SMS), 1, 1), units))
    return out


def _pack_launches(N, H, rules):
    """bffc_kf_pack, bffc_kf_pack_rfft (the same grid), bffc_dkf_unpack, bffc_dkf_unpack_half"""
    NE = _ne(N)
    R0, R1 = OUTER.get(N, (1, 1))
    R = NE // 8192
    out = []
    for hc in ([H] if rules == 'parent' else _groups(H, GRID_YZ)):
        if R0 >= 32:
            out.append(('kf_pack', (8192 // 2 // 32, (R0 // 32) * R1, hc), None))
        else:
            out.append(('kf_pack', (min((NE // 4 + 255) // 256, 32), hc, 1), None))
        if N < 8192:
            out += [('dkf_unpack', (8192 // 256, hc, 1), None), ('dkf_unpack_half', (8192 // 2 // 256 + 1, hc, 1), None)]
        else:
            out += [('dkf_unpack', (64, hc, 1), None), ('dkf_unpack_half', (1 if R < 32 else R // 32, 256, hc), None)]
    return out


def _pair_bytes(N):
    return 2 * (N // 8192 // 2 + 1) * 8192 * 8            # filter_pair_bytes


def _recommended_workspace(N, H):
    """bffc_filter_workspace_bytes"""
    per = _pair_bytes(N)
    return min((H + 1) // 2, max((576 << 20) // per, 1)) * per


def _filter_launches(N, H, workspace_bytes, rules):
    """bffc_kf_from_filter and bffc_dk_from_dkf (the same grids, mirrored)"""
    if N <= 8192:
        return [('kf_from_filter', ((H + 1) // 2, 1, 1), None), ('dk_from_dkf', (H, 1, 1), None)]
    R = N // 8192
    pairs = workspace_bytes // _pair_bytes(N)
    cap = (H + 1) // 2 if rules == 'parent' else min((H + 1) // 2, (GRID_YZ - 1) // 2)
    group = min(pairs, cap) * 2
    out = []
    for hc in _groups(H, group):
        out += [('filter cols', (R, (hc + 1) // 2, 1), None), ('filter rows', (R // 2 + 1, hc, 1), None)]
    return out


def _filter_launch_count(N, H, workspace_bytes):
    """launches of one bffc_kf_from_filter or bffc_dk_from_dkf call: one, or two per channel group"""
    if N <= 8192:
        return 1
    group = min(workspace_bytes // _pair_bytes(N), (H + 1) // 2, (GRID_YZ - 1) // 2) * 2
    return 2 * -(-H // group)


def _all_launches(N, B, H, rules):
    """every launch of every entry point at (N, B, H), tagged with the entry point"""
    out = []
    for gated, backward in itertools.product((False, True), (False, True)):
        tag = ('bwd' if backward else 'fwd') + (' gated' if gated else '')
        out += [(tag, *l) for l in _conv_launches(N, B, H, gated, backward, rules)]
    out += [('pack', *l) for l in _pack_launches(N, H, rules)]
    out += [('filter, recommended workspace', *l) for l in _filter_launches(N, H, _recommended_workspace(N, H), rules)]
    big = -(-H // 2) * _pair_bytes(N) if N > 8192 else 0        # room for every channel pair in one group
    out += [('filter, whole-H workspace', *l) for l in _filter_launches(N, H, big, rules)]
    return out


def _violations(rules):
    bad = []
    for N, B, H in itertools.product(SIZES, EXTENTS, EXTENTS):
        fits = B * H * N * 2 <= DEVICE_BYTES
        for entry, name, (x, y, z), units in _all_launches(N, B, H, rules):
            if not (1 <= x <= GRID_X and 1 <= y <= GRID_YZ and 1 <= z <= GRID_YZ):
                bad.append((N, B, H, entry, name, (x, y, z)))
            elif units is not None and fits and units > INT_MAX:
                bad.append((N, B, H, entry, name, ('units', units)))
    return bad


# ----------------------------------------------------------------------------- tests
def test_every_launch_within_grid_limits():
    bad = _violations('now')
    assert not bad, f'{len(bad)} launches exceed a grid limit, e.g. {bad[:5]}'


def _item(v):
    """which of items 1-3 of the module docstring a parent-rule violation is, or None"""
    N, B, H, entry, name, grid = v
    if name.startswith('cc level 0') and N == 16 * K and entry.startswith('fwd') and (H >= 65536 and B <= 2 or B >= 131071):
        return 1
    if name.startswith(('kf_pack', 'dkf_unpack')) and H >= 65536:
        return 2
    if entry == 'filter, whole-H workspace' and name.startswith('filter') and N > 8192 and H >= 65536:
        return 3
    return None


def test_parent_rules_fail_at_items_1_to_3():
    bad = _violations('parent')
    other = [v for v in bad if _item(v) is None]
    assert not other, f'the parent rules fail outside items 1-3: {other[:5]}'
    assert {_item(v) for v in bad} == {1, 2, 3}
    # item 1 is exactly the 16K forward: B <= 2 with H >= 65536, or B >= 131071, gated or not, plain and short kernels
    want = {(B, H) for B, H in itertools.product(EXTENTS, EXTENTS) if (B <= 2 and H >= 65536) or B >= 131071}
    assert {(v[1], v[2]) for v in bad if _item(v) == 1} == want
    assert {(v[3], v[4]) for v in bad if _item(v) == 1} == {
        (e, n) for e in ('fwd', 'fwd gated') for n in ('cc level 0', 'cc level 0 short')}
    # item 2 at every size; item 3 at every composite size, and never with the recommended workspace
    assert {v[0] for v in bad if _item(v) == 2} == set(SIZES)
    assert {v[0] for v in bad if _item(v) == 3} == {N for N in SIZES if N > 8192}


@pytest.mark.parametrize('N', [n for n in SIZES if n > 8192])
def test_chunks_below_the_cap_keep_their_geometry(N):
    """the cap changes nothing for shapes below it: the same chunk, the same count"""
    for B, H in itertools.product([1, 2, 3, 8, 259, 65535, 131070], [1, 64, 683, 4097, 65535]):
        for sets in (_nlev(N), _nlev(N) + 1):
            assert _chunk_view(N, B, H, sets) == _chunk_view(N, B, H, sets, cap=None), (N, B, H, sets)


def test_16k_forward_chunks():
    """the chunks the cap introduces at 16K forward (nlev = 1): 65535 channels or 65535 pairs, ragged tails"""
    assert _chunk_view(16 * K, 1, 65600, 1) == (1, 65535)
    assert _chunk_shapes(16 * K, 1, 65600, 1, 'now') == (2, [(1, 65)] + [(1, 65535)])
    assert _chunk_view(16 * K, 131078, 1, 1) == (131070, 1)
    assert _chunk_shapes(16 * K, 131078, 1, 1, 'now') == (2, [(8, 1), (131070, 1)])
    # the backward (two sets) was already below the cap: unchanged
    assert _chunk_view(16 * K, 1, 65600, 2) == _chunk_view(16 * K, 1, 65600, 2, cap=None) == (1, 32768)
    assert _chunk_view(16 * K, 131078, 1, 2) == _chunk_view(16 * K, 131078, 1, 2, cap=None) == (65536, 1)
