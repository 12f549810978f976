"""CPU model of how a deterministic plan (BFFC_PLAN_DETERMINISTIC) sums the filter gradient's spectrum dk_f (no GPU
needed).  The rule is csrc/dkf_slabs.cuh; launch_dkf, dkf_partial_bytes and bffc_workspace_bytes_ex / _blocked (csrc/bffc.cu) apply
it to the launches of one backward call, which are those of tests/dkf_split_model.py:

* seqlen <= 8192: one launch, rows = channels, pairs = 8192-point units per channel (2 * 8192 / seqlen members each);
* overlap-save blocks: one launch, the B * nblk blocks are the items;
* composite sizes: one launch per chunk of for_each_chunk, rows = the chunk's channels * seqlen / 8192, pairs = its batch
  pairs; a chunk whose first member is not 0 adds into the rows an earlier chunk wrote.

A row's pairs are cut into S = min(pairs, ceil(SLAB_TARGET / rows)) slabs, CTA i of a grid g takes the slabs
[n i / g, n (i + 1) / g) of the n = rows * S, and a slab's sum goes to dk_f (S = 1) or to a 64 KB partial slot (S > 1).
"""
from test_chunked_gpu import _chunk_view, _chunks, _nlev, _workspace_bytes

INNER = 8192
SLAB_TARGET = 512                 # kSlabTarget
SLOT_BYTES = INNER * 8            # one dk_f row, 8192 complex fp32


def slabs(rows, pairs):
    return min(pairs, -(-SLAB_TARGET // rows))


def slab_begin(pairs, S, s):
    return pairs * s // S


def slab_of(pairs, S, pr):
    return ((pr + 1) * S - 1) // pairs


def cta_slab(n, i, grid):
    return n * i // grid


def slab_unit(pairs, S, j):
    return (j // S) * pairs + slab_begin(pairs, S, j % S)


def partial_slots(rows, pairs):
    S = slabs(rows, pairs)
    return rows * S if S > 1 else 0


def flushes(rows, pairs, grid):
    """(row, slab, first pair, end pair) of every sum the CTAs of a grid-CTA launch store, in CTA order"""
    S = slabs(rows, pairs)
    n = rows * S
    out = []
    for i in range(grid):
        begin, end = slab_unit(pairs, S, cta_slab(n, i, grid)), slab_unit(pairs, S, cta_slab(n, i + 1, grid))
        start = begin
        for g in range(begin, end):            # the kernel's loop: a flush where a slab, a row or the range ends
            r, pr = divmod(g, pairs)
            if pr == pairs - 1 or g == end - 1 or slab_of(pairs, S, pr) != slab_of(pairs, S, pr + 1):
                out.append((r, slab_of(pairs, S, pr), start - r * pairs, pr + 1))
                start = g + 1
    return out


def launches(seqlen, B, H, L=None, halo=None):
    """(rows, pairs, accumulate) of every dk_f launch of one backward call, in launch order"""
    if halo is not None:
        items = B * -(-L // (INNER - halo))
        return [(H, (items + 1) // 2, False)]
    if seqlen <= INNER:
        members = 2 * (INNER // seqlen)
        return [(H, -(-B // members), False)]
    R = seqlen // INNER
    return [(ch * R, (cb + 1) // 2, b0 > 0) for b0, cb, _, ch in _chunks(seqlen, B, H, _nlev(seqlen) + 1)]


def partial_bytes(seqlen, B, H, L, halo=None):
    """dkf_partial_bytes: the slots of the largest launch of a call (halo: overlap-save blocks)"""
    if seqlen <= INNER:
        items = B if halo is None else B * -(-L // (INNER - halo))
        members = 2 * (INNER // seqlen)
        return partial_slots(H, -(-items // members)) * SLOT_BYTES
    R = seqlen // INNER
    cb, ch = _chunk_view(seqlen, B, H, _nlev(seqlen) + 1)
    return max(partial_slots(vh * R, (vb + 1) // 2) for vb in (cb, B % cb) for vh in (ch, H % ch) if vb and vh) * SLOT_BYTES


def _align256(n):
    return (n + 255) // 256 * 256


def default_workspace(seqlen, B, H, L, gated):
    """bffc_workspace_bytes_ex(..., backward = 1) of a default plan"""
    if seqlen <= INNER:
        return 2 * _align256(B * H * L * 2) if gated else 0
    return _workspace_bytes(seqlen, B, H, True)


def workspace_bytes(seqlen, B, H, L, gated, halo=None):
    """bffc_workspace_bytes_ex (halo None) or bffc_workspace_bytes_blocked(..., backward = 1) of a deterministic plan:
    the partial slots after the default need"""
    base, part = default_workspace(seqlen, B, H, L, gated), partial_bytes(seqlen, B, H, L, halo)
    return _align256(base) + part if part else base


def extra_launches(seqlen, B, H, L=None, halo=None):
    """launches a deterministic backward adds: one slot sum per dk_f launch with S > 1"""
    return sum(slabs(rows, pairs) > 1 for rows, pairs, _ in launches(seqlen, B, H, L, halo))
