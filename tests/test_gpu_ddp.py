"""Hardware data-parallel correctness (SURVEY §4 / §8e; VERDICT r1 weak #11): two ranks over NCCL, one process per GPU.

  * rank-sharded CUDA gradients, averaged by e2_tts_pytorch_b200.GradSync (one flat ncclAllReduce) == the single-rank gradients on the
    concatenated batch — eager step and GraphedTrainStep;
  * a step where ONE rank drops the text (trainer.py:155 `find_unused_parameters=True` semantics): the text-stream parameters get no
    gradient on that rank, the exchange still works and averages in zeros for it.
Needs 2 GPUs: run with `python -m pytest tests/test_gpu_ddp.py -m gpu` on a machine with two; skipped on a 1-GPU machine.
"""
import os
import socket
import traceback

import pytest
import torch

pytestmark = pytest.mark.gpu

TKW = dict(dim=128, depth=2, heads=2, dropout=0.0)
B, N = 4, 96


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _make(pkg, dev):
    torch.manual_seed(123)
    model = pkg.E2TTS(transformer=dict(max_seq_len=256, **TKW), use_vocos=False)
    from oracle import e2tts_oracle as O
    model.load_state_dict(O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=7))
    model.to(dev).train()
    model.cond_drop_prob = 0.0
    return model


def _data(dev):
    g = torch.Generator().manual_seed(5)
    mel = torch.randn(B, N, 100, generator=g)
    x0 = torch.randn(B, N, 100, generator=g)
    times = torch.rand(B, generator=g)
    span = torch.zeros(B, N, dtype=torch.bool)
    for b in range(B):
        span[b, 10 + 3 * b: 60 + 3 * b] = True          # the same number of masked frames on every sample: mean of rank means == global mean
    return mel.to(dev), x0.to(dev), times.to(dev), span.to(dev)


def _grads_of(pkg, model, sl, data, text, drop):
    mel, x0, times, span = data
    for p in model.parameters():
        p.grad = None
    with pkg.inject_randomness(x0=x0[sl], times=times[sl], span_mask=span[sl], drop_text_cond=drop):
        out = model(mel[sl], text=text[sl])
    out.loss.backward()
    return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in model.named_parameters()}, float(out.loss)


def _worker(rank, world, port, errs):
    try:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        import torch.distributed as dist
        import e2_tts_pytorch_b200 as pkg
        torch.cuda.set_device(rank)
        dev = torch.device('cuda', rank)
        dist.init_process_group('nccl', device_id=dev)
        model = _make(pkg, dev)
        # replicas must be identical: the hyper-connections' initial stream is drawn with python's randrange (rank dependent)
        sa = model.transformer.hyper_conns[0][0][0].static_alpha.detach().clone()
        pkg.broadcast_module(model)
        gathered = [torch.zeros_like(sa) for _ in range(world)]
        dist.all_gather(gathered, model.transformer.hyper_conns[0][0][0].static_alpha.detach())
        assert all(torch.equal(g, gathered[0]) for g in gathered)
        data = _data(dev)
        text = pkg.list_str_to_tensor(['Hello', 'Goodbye', 'Good morning', 'Hi']).to(dev)
        mine = slice(2 * rank, 2 * rank + 2)
        names = [n for n, _ in model.named_parameters()]

        # ---- what the exchange must produce, computed locally on every rank from the full data
        g_all, _ = _grads_of(pkg, model, slice(0, B), data, text, False)
        g_r0, _ = _grads_of(pkg, model, slice(0, 2), data, text, False)
        g_r1, _ = _grads_of(pkg, model, slice(2, 4), data, text, False)
        g_r0_drop, _ = _grads_of(pkg, model, slice(0, 2), data, text, True)
        text_params = [n for n in names if g_r0_drop[n] is None]
        assert len(text_params) > 20 and all(('.1.' in n or 'text' in n) for n in text_params), text_params[:5]

        # ---- 1. eager step + GradSync == single-rank gradients on the concatenated batch
        sync = pkg.GradSync(list(model.parameters()))
        assert sync.world == world
        _grads_of(pkg, model, mine, data, text, False)      # leaves this rank's gradients in p.grad
        sync()
        for n, p in model.named_parameters():
            want = g_all[n]
            if float(want.norm()) > 0:
                assert _rel(p.grad, want) < 5e-3, ('eager', n, _rel(p.grad, want))
        assert float(sync.used.min()) == float(world)

        # ---- 2. one rank drops the text: zeros are averaged in for its text-stream parameters
        _grads_of(pkg, model, mine, data, text, rank == 0)
        assert (model.transformer.text_registers.grad is None) == (rank == 0)
        sync()
        for n, p in model.named_parameters():
            a = g_r0_drop[n]
            want = 0.5 * ((a if a is not None else torch.zeros_like(g_r1[n])) + g_r1[n])
            if float(want.norm()) > 0:
                assert _rel(p.grad, want) < 5e-3, ('drop', n, _rel(p.grad, want))
        used = dict(zip(names, sync.used.tolist()))
        assert all(used[n] == 1.0 for n in text_params) and used['to_pred.weight'] == 2.0

        # ---- 3. GraphedTrainStep: graph replay + ONE flat all-reduce
        for p in model.parameters():
            p.grad = None
        mel, x0, times, span = data
        with pkg.inject_randomness(x0=x0[mine], times=times[mine], span_mask=span[mine], drop_text_cond=False):
            step = pkg.GraphedTrainStep(model, mel[mine].contiguous(), text=text[mine].contiguous())
            assert step.grad_sync is not None and step.grad_sync.world == world
            loss = float(step())
        for n, p in model.named_parameters():
            want = g_all[n]
            if float(want.norm()) > 0:
                assert _rel(p.grad, want) < 5e-3, ('graph', n, _rel(p.grad, want))
        assert loss == loss
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        errs.put((rank, traceback.format_exc()))
        raise


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_rank_gradients_match_single_rank_on_concatenated_batch():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    errs = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, errs)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    msgs = []
    while not errs.empty():
        msgs.append(errs.get())
    for p in procs:
        if p.is_alive():
            p.kill()
            msgs.append((-1, 'worker timed out'))
    assert not msgs and all(p.exitcode == 0 for p in procs), '\n'.join(f'rank {r}:\n{m}' for r, m in msgs)
