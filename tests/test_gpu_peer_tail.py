"""dist.PeerTail: the training-step tail (gradient exchange -> TV -> MaskedAdam) as ONE sweep over peer-mapped memory.

world = 1 (any GPU box): bit-identical to total_variation_add_grad + MaskedAdam.step(), persistent gradient buffers filled by the
march backward, a short training run.  world = 2 (needs two GPUs; skipped on a one-GPU box): two NCCL ranks with DIFFERENT
synthetic gradients must end up, on both ranks, with exactly the parameters a single process computes from the mean gradient --
this pins ownership ranges, P2P loads / stores, the ping-pong swap and both barriers.  The fixed summation order makes it exact."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _model(seed=3, world=20, F_=2):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    return models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=world ** 3, num_voxels_base_density=world ** 3,
                                   num_voxels_rgb=world ** 3, num_voxels_base_rgb=world ** 3, num_voxels_viewdir=-1, alpha_init=1e-4,
                                   fast_color_thres=0, rgbnet_dim=12, fourier_freq_num=F_)


def _opt(m):
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    return create_optimizer_or_freeze_model(m, dict(lrate_density=0.1, lrate_k0=0.1, lrate_rgbnet=1e-3, lrate_decay=20,
                                                    skip_zero_grad_fields=['density', 'k0']), 0)


def _synthetic_grads(m, seed, dev):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, p in m.named_parameters():
        if p.requires_grad:
            out[name] = (torch.randn(p.shape, generator=g) * (torch.rand(p.shape, generator=g) > 0.5)).to(dev)
    return out


def _set_grads(m, grads):
    for name, p in m.named_parameters():
        if name not in grads:
            continue
        buf = getattr(p, '_ubn_grad_buffer', None)
        if buf is not None:
            buf.copy_(grads[name])
            p.grad = buf
        else:
            p.grad = torch.empty_like(p, memory_format=torch.preserve_format).copy_(grads[name])


def test_peer_tail_world1_is_bit_identical_to_tv_then_step():
    from unboundednerfpytorch_b200 import dist as D
    ma, mb = _model().to(DEV), _model().to(DEV)
    oa, ob = _opt(ma), _opt(mb)
    tail = D.PeerTail(ob)
    assert mb.k0.grid in tail.grids and mb.density.grid not in tail.grids      # 12-channel grid: peer route, C = 1: classic
    assert mb.k0.grid.stride() == ma.k0.grid.stride()
    for it in range(3):
        grads = _synthetic_grads(ma, 100 + it, DEV)
        _set_grads(ma, grads)
        _set_grads(mb, grads)
        dense = it != 1
        ma.density_total_variation_add_grad(1e-3, dense)
        ma.k0_total_variation_add_grad(1e-4, dense)
        oa.step()
        tail.step(mb.tv_terms(1e-3, 1e-4, dense))
        for (ka, va), (kb, vb) in zip(ma.state_dict().items(), mb.state_dict().items()):
            assert ka == kb and torch.equal(va, vb), f'{ka} differs after step {it}'
        for pa, pb in zip(ma.parameters(), mb.parameters()):
            if pa.requires_grad:
                assert torch.equal(oa.state[pa]['exp_avg'], ob.state[pb]['exp_avg'])
                assert torch.equal(oa.state[pa]['exp_avg_sq'], ob.state[pb]['exp_avg_sq'])
        assert mb.k0.grid.grad is None and float(mb.k0.grid._ubn_grad_buffer.abs().max()) == 0.0      # consumed and re-zeroed


def test_march_backward_fills_the_persistent_buffer_and_training_works():
    from tests.util import seeded_rays
    from unboundednerfpytorch_b200 import dist as D
    ma, mb = _model(seed=5, world=24).to(DEV), _model(seed=5, world=24).to(DEV)
    with torch.no_grad():
        for m in (ma, mb):
            m.density.grid.normal_(0, 1, generator=torch.Generator(device=DEV).manual_seed(1))
            m.k0.grid.normal_(0, 1, generator=torch.Generator(device=DEV).manual_seed(2))
    oa, ob = _opt(ma), _opt(mb)
    tail = D.PeerTail(ob)
    ro, rd, vd = seeded_rays(512, 9, DEV)
    target = torch.rand(512, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5)
    la, lb = [], []
    for it in range(1, 6):
        for m, opt, losses in ((ma, oa, la), (mb, ob, lb)):
            out = m(ro, rd, vd, global_step=it, is_train=True, **rk)
            opt.zero_grad(set_to_none=True)
            loss = torch.nn.functional.mse_loss(out['rgb_marched'], target)
            loss.backward()
            losses.append(loss.item())
            if m is mb:
                assert m.k0.grid.grad is m.k0.grid._ubn_grad_buffer         # the scatter went straight into the persistent buffer
                tail.step(m.tv_terms(1e-6 / 512, 1e-7 / 512, True))
            else:
                m.density_total_variation_add_grad(1e-6 / 512, True)
                m.k0_total_variation_add_grad(1e-7 / 512, True)
                opt.step()
    assert lb[-1] < lb[0]
    # same training trajectory up to the atomics' summation order (Adam turns last-bit gradient differences into visible ones
    # only where g ~ 0, i.e. on parameters that barely matter for the loss)
    assert all(abs(a - b) <= 1e-4 * abs(a) for a, b in zip(la, lb)), (la, lb)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from unboundednerfpytorch_b200 import dist as D
    try:
        D.init_from_env()
        dev = torch.device('cuda', rank)
        torch.cuda.set_device(dev)
        m = _model().to(dev)                                  # same seed on every rank: identical replicas
        opt = _opt(m)
        tail = D.PeerTail(opt)
        want = _model().to(dev)                               # single-process restatement on this rank: mean gradient -> TV -> step
        wopt = _opt(want)
        for it in range(3):
            per_rank = [_synthetic_grads(m, 1000 * it + r, dev) for r in range(world)]
            _set_grads(m, per_rank[rank])
            mean = {}
            for k in per_rank[0]:
                s = per_rank[0][k].clone()
                for r in range(1, world):
                    s = s + per_rank[r][k]                    # rank order, like the kernel
                mean[k] = s * (1.0 / world)
            _set_grads(want, mean)
            dense = it != 1
            want.density_total_variation_add_grad(1e-3, dense)
            want.k0_total_variation_add_grad(1e-4, dense)
            wopt.step()
            tail.step(m.tv_terms(1e-3, 1e-4, dense))
            torch.cuda.synchronize()
            sd_want, sd_ours = want.state_dict(), m.state_dict()
            # the peer kernel sums the ranks' gradients in rank order, like `mean` above: exact
            assert torch.equal(sd_want['k0.grid'], sd_ours['k0.grid']), \
                f"rank {rank}: k0.grid differs after step {it}: {(sd_want['k0.grid'] - sd_ours['k0.grid']).abs().max().item():.3e}"
            for ka, va in sd_want.items():
                if ka.startswith(('density.grid', 'rgbnet')):
                    # classic route: NCCL's mean all-reduce.  For more than two ranks its summation order is not ours, and Adam's
                    # m / sqrt(v) turns a last-bit difference of a near-zero mean gradient into a full +-lr step: judged by the
                    # fraction of elements that moved apart, not element by element
                    vb = sd_ours[ka]
                    bad = ((va - vb).abs() > 1e-6 + 1e-5 * va.abs()).float().mean().item()
                    assert bad <= (0.0 if world == 2 else 2e-3), \
                        f'rank {rank}: {ka}: {bad:.2e} of the elements differ after step {it} (max {(va - vb).abs().max().item():.3e})'
        tail.gather_moments()
        full = opt.state[m.k0.grid]['exp_avg']
        assert torch.equal(full, wopt.state[want.k0.grid]['exp_avg']), 'gathered exp_avg differs'
        q.put((rank, 'ok'))
    except Exception:
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 4, 8])
def test_peer_tail_ranks_nccl_match_single_process_mean_gradient_step(world):
    """world NCCL ranks (one per GPU of the box; skipped where the box has fewer) fed DIFFERENT synthetic gradients must end up with
    exactly the parameters and moments a single process computes from the mean gradient: k_tv_adam_peer<2 / 4 / 8>."""
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    assert sorted(res) == [(r, 'ok') for r in range(world)], res
