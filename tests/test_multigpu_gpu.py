"""Multi-rank parity on real GPUs: `parallel.sharded_conv(FlashFFTConv ...)` under NCCL with one process per GPU —
each rank convolves its channel block, the blocks are all-gathered over NVLink, every rank checks the full output
against the oracle.  Skipped when fewer than 2 GPUs are visible (the driver's GPU test box has one)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, N, B, H, L, gated, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, 'flash-fft-conv_b200'))
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import FlashFFTConv, parallel
    from oracle import fftconv_oracle as orc
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    d = orc.make_inputs(B, H, N, L, torch.bfloat16, seed=17, gated=gated, unit_scale=True)
    conv = FlashFFTConv(N, dtype=torch.bfloat16).cuda()
    gates = (d['pregate'].cuda(), d['postgate'].cuda()) if gated else ()
    y = parallel.sharded_conv(lambda *a: conv(*a), d['u'].cuda(), d['k'].cuda(), gates=gates)
    ref = orc.ref_fft_conv_gated(d['u'], d['k'], d['pregate'], d['postgate'], N) if gated else orc.ref_fft_conv(d['u'], d['k'], N)
    rel = ((y.float().cpu() - ref.float()).norm() / ref.float().norm()).item()
    # backward on the local channel block: dk of the block needs no reduction (sum over b is local)
    h0, h1 = parallel.channel_range(H, world, rank)
    ul, kl = d['u'][:, h0:h1].contiguous().cuda().requires_grad_(True), d['k'][h0:h1].contiguous().cuda().requires_grad_(True)
    conv(ul, kl).backward(d['dout'][:, h0:h1].contiguous().cuda())
    _, dk_ref = orc.ref_grads(d['u'][:, h0:h1], d['k'][h0:h1], d['dout'][:, h0:h1], N)
    rel_dk = ((kl.grad.cpu() - dk_ref).norm() / dk_ref.norm()).item()
    q.put((rank, rel, rel_dk))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
@pytest.mark.parametrize('N,B,H,L,gated', [(8192, 4, 10, 8192, False), (32768, 2, 6, 16384, True), (1048576, 2, 4, 1048576, False)])
def test_sharded_conv_nccl(N, B, H, L, gated):
    world = min(torch.cuda.device_count(), 4)
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, N, B, H, L, gated, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
    for rank, rel, rel_dk in res:
        assert rel <= 1e-2, (rank, rel)
        assert rel_dk <= 1e-2, (rank, rel_dk)
