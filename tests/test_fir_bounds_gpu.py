"""GPU tests of the short explicit filters element by element (fir_conv, fir_mixer, with and without docs=;
csrc/fir_conv.cuh).  Run with `-m gpu` on an H100.

Every output element of y, du, dpregate and dpostgate is bounded against tests/fir_model.py's fp64 direct lag sums,

    |got - ref| <= ulp_dt(ref) + C * 2^-24 * mag,

and every lag of dk by |got - ref| <= C_DK * dk_depth * 2^-24 * mag; an output (or lag) whose terms all read zero is
exactly 0.  Inputs are uniform samples scaled per 64-sample block by 2^j with some blocks all zero
(fir_model.block_scaled), so that a read past L, from the neighbouring (member, channel) row or from another document
shows at the element it lands on, which a rel-L2 per row would dilute.

1. Every tap count: Lk = 1 .. 128, bf16 and fp16, ungated and gated, G in {H, 1}, B = 2, H = 16, L = 4096 + 64 + 40
   (two tiles, the second ragged, L not a multiple of 64): every (P, dk skip mask) class of the kernels.
2. Short rows: L in {1, 7, 8, 9, 63, 64, 65, Lk - 1, Lk, Lk + 1} at LKS_COVER (one Lk or more of every class, every
   dk_pairs lag-slot bucket): the zero padding to a multiple of 8 and the trim back to L.
3. Tile and slab edges: B = 3, L = 2 * 65536 + 4096 + 24 (two full slabs of 16 tiles and a ragged third), gated, at
   LKS_COVER.
4. fir_mixer in place at L = 4096 + 24 (read in place) and 4096 + 21 (padded): y, every slice of the (B, 3D, L)
   gradient and dk.
5. docs=: the masked model (a lag counts within its document only) at LKS_DOCS (LKS_COVER and every dk_pairs slot
   edge), on hand-built layouts (a boundary at every residue of its 64-sample block; boundaries 0, 1, 64P - 1, 64P and
   64P + 1 samples before and after a tile edge and a slab edge; documents of length 1, Lk - 1, Lk and Lk + 1;
   several boundaries in one block; a document spanning a whole tile; a ragged L) and seeded make_cu layouts.  The
   statistic is kept apart for the dirty rows (test_fir_docs.marked_rows: fmaf in ascending lag order on the CUDA
   cores) and the clean ones (the tensor cores' MMA sums).
6. Negative control: one element of a real output moved by 0.3 of its row's rms, at a tile edge of case 3 and at a
   document boundary of case 5, is flagged by the bound, and no other element is.

Largest statistics, max over elements of (|got - ref| - ulp) / (2^-24 mag) (dk: |got - ref| / (dk_depth 2^-24 mag)),
per (dtype, quantity, path), measured on an H100 80GB HBM3 at a 700 W power limit ($BFFC_FIR_BOUNDS_TABLE, if set,
receives them as JSON after the module).  plain: cases 1-4 (L = 4200 unless stated); docs clean / dirty: case 5's
tensor-core and CUDA-core rows.

    quantity  path        bf16                                      fp16
    y         plain       0.641   Lk=124 G=1 ungated                1.43    Lk=115 G=16 gated
    y         docs clean  0.300   tile_slab_edges Lk=128 gated      1.72    tile_slab_edges Lk=127 gated
    y         docs dirty  0.184   residues Lk=9 ungated             0.766   tile_slab_edges Lk=32 gated
    du        plain       0.825   Lk=127 G=1 gated                  1.72    Lk=114 G=16 ungated
    du        docs clean  0.283   tile_slab_edges Lk=65 gated       0.845   whole_tile Lk=127 gated
    du        docs dirty  0.0288  tile_slab_edges Lk=127 gated      0.318   residues Lk=113 gated
    dpregate  plain       0.885   Lk=127 G=1 gated                  0.875   Lk=110 G=16 gated
    dpregate  docs clean  2.18    tile_slab_edges Lk=89 gated       0.865   whole_tile Lk=127 gated
    dpregate  docs dirty  0.0154  tile_slab_edges Lk=127 gated      0.488   residues Lk=113 gated
    dpostgate plain       0.369   Lk=80 G=1 gated                   1.31    Lk=115 G=16 gated
    dpostgate docs clean  0.385   tile_slab_edges Lk=64 gated       1.53    tile_slab_edges Lk=127 gated
    dpostgate docs dirty  0.198   tile_slab_edges Lk=64 gated       0.790   tile_slab_edges Lk=32 gated
    dk        plain       0.0375  Lk=102 G=16 gated                 0.0305  Lk=88 G=16 gated
    dk        docs        0.00587 lengths Lk=8 ungated              0.00442 lengths Lk=18 gated

C = 6.5 and C_DK = 0.12 are about 3x the largest of them.  The worst elements are interior samples of tensor-core rows
whose terms cancel (|ref| 1e-6 to 1e-4 of mag), not edges.  The statistic grows with the MMA steps an output
accumulates: over case 1's gated runs at G = H its maximum is 0 at P = 0, 0.55 at P = 1 and 1.43 at P = 2.  fp16
shows it more than bf16 because its output ulp is 8x finer.  The CUDA-core rows (fmaf, round to nearest) stay lower.
The module took 54 s on that H100.
"""
import json
import os

import pytest
import torch

from fir_model import BLOCK, SLAB_TILES, TILE, bound_inputs, dk_depth, dk_excess, excess, model, p_of, segments
from test_fir_docs import boundaries, marked_rows
from varlen_oracle import make_cu

pytestmark = pytest.mark.gpu

DEV = 'cuda'
C = 6.5
C_DK = 0.12
DTYPES = [torch.bfloat16, torch.float16]
SLAB = TILE * SLAB_TILES

LKS_ALL = list(range(1, 129))
# one Lk or more of each of the 17 (P, dk skip mask) classes, and of the five dk_pairs lag-slot buckets
# (test_fir_bounds.py checks that they still are)
LKS_COVER = [1, 2, 9, 10, 18, 33, 41, 42, 50, 64, 65, 66, 81, 89, 97, 98, 113, 114, 127, 128]
LKS_DOCS = sorted(set(LKS_COVER) | {8, 16, 17, 32, 33})

# largest statistic per (dtype, quantity, path) with its case; written to $BFFC_FIR_BOUNDS_TABLE, if set
STATS = {}


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()
    yield
    if os.environ.get('BFFC_FIR_BOUNDS_TABLE'):
        with open(os.environ['BFFC_FIR_BOUNDS_TABLE'], 'w') as f:
            json.dump({' '.join(k): v for k, v in sorted(STATS.items())}, f, indent=1)


def record(key, value, case):
    if value > STATS.get(key, (-1.0, ''))[0]:
        STATS[key] = (value, case)


def run(u, k, pre, post, dout, docs=None):
    """{name: output} of fir_conv forward and backward"""
    from flashfftconv import fir_conv
    u = u.clone().requires_grad_(True)
    k = k.clone().requires_grad_(True)
    gates = ()
    if pre is not None:
        pre, post = pre.clone().requires_grad_(True), post.clone().requires_grad_(True)
        gates = (pre, post)
    y = fir_conv(u, k, pre, post, docs=docs)
    y.backward(dout)
    out = {'y': y.detach(), 'du': u.grad, 'dk': k.grad}
    if gates:
        out['dpre'], out['dpost'] = pre.grad, post.grad
    return out


def excesses(got, ref, dt, B, gs, L, Lk, docs=False):
    """{name: per-element excess} of the outputs and dk (dk: over dk_depth), and whether every output or lag whose
    terms all read zero is exactly 0"""
    ex, zero = {}, True
    for name, (r, mag) in ref.items():
        a = got[name]
        if name == 'dk':
            ex[name] = dk_excess(a, r, mag, dk_depth(B, gs, L, Lk, docs))
        else:
            ex[name] = excess(a, r, mag, dt)
        zero = zero and bool((a[mag == 0] == 0).all())
    return ex, zero


def check(got, ref, dt, case, B, gs, L, Lk, dirty=None):
    """Record the statistics, then assert the bounds.  dirty: the document kernels' CUDA-core rows, {'f': forward,
    'b': backward} (B, 1, L) masks: forward-dirty rows give y and dpostgate, backward-dirty rows du and dpregate."""
    dn = 'bf16' if dt == torch.bfloat16 else 'fp16'
    ex, zero = excesses(got, ref, dt, B, gs, L, Lk, docs=dirty is not None)
    worst = {}
    for name, e in ex.items():
        worst[name] = e.max().item()
        if name == 'dk':
            record((dn, name, 'plain' if dirty is None else 'docs'), worst[name], case)
        elif dirty is None:
            record((dn, name, 'plain'), worst[name], case)
        else:
            d = dirty['f' if name in ('y', 'dpost') else 'b']
            record((dn, name, 'docs clean'), e.masked_fill(d, 0).max().item(), case)
            record((dn, name, 'docs dirty'), e.masked_fill(~d, 0).max().item(), case)
    assert zero, ('an output of zero terms is not 0', case)
    for name, s in worst.items():
        assert s <= (C_DK if name == 'dk' else C), (name, case, s)


# ------------------------------------------------------------------------------------------------ 1. every tap count
@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', LKS_ALL)
def test_every_tap_count(Lk, dt, gated):
    B, H, L = 2, 16, TILE + BLOCK + 40
    for G in (H, 1):
        u, k, pre, post, dout = bound_inputs(B, H, L, Lk, G, dt, gated, seed=Lk * 4 + G, device=DEV)
        check(run(u, k, pre, post, dout), model(u, k, pre, post, dout), dt, f'L={L} Lk={Lk} G={G} gated={gated}',
              B, H // G, L, Lk)


# ------------------------------------------------------------------------------------------------ 2. short rows
@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', LKS_COVER)
def test_short_rows(Lk, dt):
    B, H, G = 2, 8, 2
    for L in sorted({1, 7, 8, 9, 63, 64, 65, Lk - 1, Lk, Lk + 1} - {0}):
        for gated in (False, True):
            u, k, pre, post, dout = bound_inputs(B, H, L, Lk, G, dt, gated, seed=Lk * 200 + L, device=DEV)
            check(run(u, k, pre, post, dout), model(u, k, pre, post, dout), dt, f'L={L} Lk={Lk} gated={gated}',
                  B, H // G, L, Lk)


# ------------------------------------------------------------------------------------------------ 3. tile, slab edges
EDGE_SHAPE = (3, 4, 2 * SLAB + TILE + 24, 2)         # B, H, L, G


def edge_case(Lk, dt):
    B, H, L, G = EDGE_SHAPE
    u, k, pre, post, dout = bound_inputs(B, H, L, Lk, G, dt, True, seed=Lk + 7, device=DEV)
    return run(u, k, pre, post, dout), model(u, k, pre, post, dout)


@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', LKS_COVER)
def test_tile_and_slab_edges(Lk, dt):
    B, H, L, G = EDGE_SHAPE
    got, ref = edge_case(Lk, dt)
    check(got, ref, dt, f'B={B} L={L} Lk={Lk}', B, H // G, L, Lk)


# ------------------------------------------------------------------------------------------------ 4. fir_mixer
@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', [10, 66, 128])
@pytest.mark.parametrize('L', [TILE + 24, TILE + 21])
def test_mixer_in_place(L, Lk, dt):
    from flashfftconv import fir_mixer
    B, D, G = 2, 16, 4
    v, k, x1, x2, dout = bound_inputs(B, D, L, Lk, G, dt, True, seed=L + Lk, device=DEV)
    x = torch.cat([x1, x2, v], 1).requires_grad_(True)
    kk = k.clone().requires_grad_(True)
    y = fir_mixer(x, kk, D)
    y.backward(dout)
    g = x.grad
    assert g.shape == x.shape and g.is_contiguous()
    got = {'y': y.detach(), 'dpre': g[:, :D], 'dpost': g[:, D:2 * D], 'du': g[:, 2 * D:], 'dk': kk.grad}
    check(got, model(v, k, x1, x2, dout), dt, f'mixer L={L} Lk={Lk}', B, D // G, L, Lk)


# ------------------------------------------------------------------------------------------------ 5. docs=
def _cu(bounds, L):
    """int32 offsets of rows of length L from each row's sorted interior boundaries"""
    cu = [0]
    for b, row in enumerate(bounds):
        cu += [b * L + c for c in sorted(set(row)) if 0 < c < L] + [(b + 1) * L]
    return torch.tensor(cu, dtype=torch.int32)


def layouts(Lk):
    """{name: (cu, B, L)} of the hand-built and seeded document layouts at Lk"""
    P = p_of(Lk)
    offs = sorted({s * d for d in (0, 1, 64 * P - 1, 64 * P, 64 * P + 1) for s in (-1, 1)})
    L = TILE + BLOCK + 40
    cuts, c = [], 0
    while c < L:                                     # documents of 1, Lk - 1, Lk and Lk + 1 samples in turn
        c += (1, Lk - 1, Lk, Lk + 1)[len(cuts) % 4]
        cuts.append(c)
    Le = SLAB + TILE + 40
    Lw = 2 * TILE + 200
    return {
        'residues': (_cu([[65 * j for j in range(1, 64)]], L), 1, L),
        'tile_slab_edges': (_cu([[TILE + d, SLAB + d] for d in offs], Le), len(offs), Le),
        'lengths': (_cu([cuts], L), 1, L),
        'one_block': (_cu([[130, 131, 133, 140, 160, 191, 192, 1000, 1001]], L), 1, L),
        'whole_tile': (_cu([[TILE - 96, 2 * TILE + 108]], Lw), 1, Lw),
        'ragged': (make_cu(2, 5003, seed=Lk), 2, 5003),
        'seeded': (make_cu(2, 6002, seed=100 + Lk), 2, 6002),
    }


def dirty_masks(cu, B, L, Lk):
    """(B, 1, L) masks of the forward- and backward-dirty rows the document kernels mark (rows of the padded Lp)"""
    Lp = (L + 7) // 8 * 8
    n_rows = -(-Lp // BLOCK)
    f = torch.zeros(B, 1, L, dtype=torch.bool, device=DEV)
    bk = torch.zeros_like(f)
    row = torch.arange(L, device=DEV) // BLOCK
    for b in range(B):
        fd, bd = marked_rows(boundaries(cu.tolist(), b, L, Lp), n_rows, p_of(Lk))
        f[b, 0] = torch.isin(row, torch.tensor(sorted(fd), dtype=torch.long, device=DEV))
        bk[b, 0] = torch.isin(row, torch.tensor(sorted(bd), dtype=torch.long, device=DEV))
    return {'f': f, 'b': bk}


def docs_case(Lk, dt, name, gated):
    from flashfftconv import DocumentTable
    cu, B, L = layouts(Lk)[name]
    H, G = 4, 2
    u, k, pre, post, dout = bound_inputs(B, H, L, Lk, G, dt, gated, seed=Lk * 31 + len(name), device=DEV)
    got = run(u, k, pre, post, dout, DocumentTable(cu, B, L))
    ref = model(u, k, pre, post, dout, seg=segments(cu, B, L, DEV))
    return got, ref, (cu, B, L, H // G)


@pytest.mark.parametrize('dt', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('Lk', LKS_DOCS)
def test_docs(Lk, dt):
    for name in layouts(Lk):
        for gated in ((True,) if name == 'tile_slab_edges' else (False, True)):
            got, ref, (cu, B, L, gs) = docs_case(Lk, dt, name, gated)
            check(got, ref, dt, f'docs {name} Lk={Lk} gated={gated}', B, gs, L, Lk, dirty_masks(cu, B, L, Lk))


# ------------------------------------------------------------------------------------------------ 6. negative control
def _flagged_alone(got, ref, dt, name, at, B, gs, L, Lk):
    """move got[name][at] by 0.3 of its row's rms: the bound flags that element and no other"""
    r = ref[name][0]
    a = got[name].double().clone()
    b, h, t = at
    a[b, h, t] += 0.3 * r[b, h].pow(2).mean().sqrt()
    ex, _ = excesses(dict(got, **{name: a}), {name: ref[name]}, dt, B, gs, L, Lk)
    bad = ex[name] > C
    return int(bad.sum()) == 1 and bool(bad[b, h, t])


def test_planted_error_is_flagged_alone():
    dt, Lk = torch.bfloat16, 66
    B, H, L, G = EDGE_SHAPE
    got, ref = edge_case(Lk, dt)
    assert _flagged_alone(got, ref, dt, 'y', (1, 2, 2 * TILE), B, H // G, L, Lk)
    assert _flagged_alone(got, ref, dt, 'du', (2, 1, SLAB), B, H // G, L, Lk)
    got, ref, (cu, B, L, gs) = docs_case(Lk, dt, 'residues', True)
    assert _flagged_alone(got, ref, dt, 'y', (0, 1, 65 * 10), B, gs, L, Lk)
    assert _flagged_alone(got, ref, dt, 'du', (0, 3, 65 * 33 - 1), B, gs, L, Lk)
