"""CPU model of how the filter gradient's spectrum dk_f is summed (no GPU needed).

dkf3_kernel (csrc/dkf3_r128.cuh) numbers its work g = row * pairs + pair, cuts [0, rows * pairs) into gridDim.x
contiguous ranges [total * i // grid, total * (i + 1) // grid), and each CTA adds its partial sum of a row to the zeroed
gradient with red.global.add.v4.f32 when the row ends or when its own range does.  launch_dkf (csrc/bffc.cu) launches
grid = min(units, SMs) CTAs.  What a row and a pair are depends on the size:

* seqlen <= 8192 (fill_seq_tiles): a row is a channel, a pair is one 8192-point unit holding 2 * 8192 / seqlen batch
  members (two at 8192), so pairs = ceil(B / members);
* overlap-save blocks (fill_blocks): the items are the B * nblk blocks of S = 8192 - halo samples, two per unit;
* composite sizes (fill_complex_rows): a channel has R = seqlen / 8192 rows of its own, one launch per chunk of
  for_each_chunk (chunk_view with nlev + 1 plane sets), pairs = the chunk's batch pairs; batch chunks of one channel
  add into the same rows, one launch after the other.

The number of additions that land on one address of dk_f is therefore the number of CTAs a row's units straddle, summed
over the batch chunks.  Floating-point addition is commutative, so up to two additions into a zero give the same bits in
either order; from three on (or two into a non-zero sum left by an earlier batch chunk) the result depends on the order
the hardware serves them in.
"""
from test_chunked_gpu import _chunks, _nlev

INNER = 8192
EXACT_FLUSHES = 2          # a + b == b + a: at most this many additions into a zero cannot depend on their order


def persistent_grid(units, num_sms, per_block=1):
    """persistent_grid (bffc.cu): one CTA per `per_block` units, at most one per SM"""
    return min(-(-units // per_block), num_sms)


def cta_ranges(total, grid):
    """[g_begin, g_end) of every CTA of dkf3_kernel"""
    return [(total * i // grid, total * (i + 1) // grid) for i in range(grid)]


def row_flushes(rows, pairs, num_sms):
    """additions into each of the `rows` dk_f rows of one dkf3_kernel launch: the CTAs whose range holds one of the
    row's units"""
    total = rows * pairs
    out = [0] * rows
    for b, e in cta_ranges(total, persistent_grid(total, num_sms)):
        if e > b:
            for r in range(b // pairs, (e - 1) // pairs + 1):
                out[r] += 1
    return out


def blocked_items(B, L, halo):
    """fill_blocks: the overlap-save blocks of a call are its batch items"""
    S = INNER - halo
    return B * -(-L // S)


def launch_flushes(seqlen, B, H, num_sms, L=None, halo=None):
    """For each channel, one entry per dkf3_kernel launch that adds into its dk_f rows (one launch, or one per batch
    chunk at a composite size): the largest number of additions of that launch into one address.
    halo: overlap-save blocks of a length-L call on the seqlen-8192 plan (bffc_bwd_blocked)."""
    if halo is not None:
        assert seqlen == INNER
        return [[n] for n in row_flushes(H, (blocked_items(B, L, halo) + 1) // 2, num_sms)]
    if seqlen <= INNER:
        members = 2 * (INNER // seqlen)
        return [[n] for n in row_flushes(H, -(-B // members), num_sms)]
    R = seqlen // INNER
    out = [[] for _ in range(H)]
    for _, cb, h0, ch in _chunks(seqlen, B, H, _nlev(seqlen) + 1):
        per_row = row_flushes(ch * R, (cb + 1) // 2, num_sms)
        for h in range(ch):
            out[h0 + h].append(max(per_row[h * R:(h + 1) * R]))
    return out


def flushes_per_channel(seqlen, B, H, num_sms, L=None, halo=None):
    """For each channel, the additions into one address of its dk_f rows in one bffc_bwd call"""
    return [sum(n) for n in launch_flushes(seqlen, B, H, num_sms, L, halo)]


def max_flushes(seqlen, B, H, num_sms, L=None, halo=None):
    return max(flushes_per_channel(seqlen, B, H, num_sms, L, halo))


def is_exact(seqlen, B, H, num_sms, L=None, halo=None):
    """True when dk must be bit-identical from run to run: launches follow each other in stream order, the first adds
    into zeros (two additions commute), a later one into what is already there (only a single addition is ordered)"""
    return all(n[0] <= EXACT_FLUSHES and all(m <= 1 for m in n[1:])
               for n in launch_flushes(seqlen, B, H, num_sms, L, halo))
