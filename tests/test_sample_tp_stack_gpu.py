"""GPU, 2 devices: DecodeStack(tp_size=2, sample=True).  Each rank's ids must equal b2_sample applied to the
concatenation of the ranks' logits shards at the same offsets, every rank's offsets must match, and the step must run the
greedy TP step's launches plus the number its docstring states; with collective "b2" both stacks' launch counts equal the
kernel nodes of a captured step.  Skipped on a machine with one GPU."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret, collective, logprobs, penalties, graph):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "dash-infer_b200", "python"))
    import torch.distributed as dist
    from b200spark import model, ops
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    B = 3
    kw = dict(wbits=4, span=16, seed=7, tp_rank=rank, tp_size=world, collective=collective, logprobs=logprobs,
              penalties=penalties)
    st = model.DecodeStack(model.TINY, B, 64, sample=True, **kw)
    greedy = model.DecodeStack(model.TINY, B, 64, **kw)
    greedy.step()
    st.set_sampling(temperature=[0.7, 1.0, 0.0], top_k=[50, 0, 0], top_p=[0.9, 1.0, 1.0], seeds=[11, 12, 13], offsets=[0, 5, 9])
    if penalties:
        st.set_penalties(repetition=1.3, presence=0.2)
        for b in range(B):
            st.set_history(b, torch.tensor([1, 2, 3 + b], dtype=torch.int32, device="cuda"))
    if graph:
        st.capture()
    ids = torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda")
    ok, msgs = True, []
    for it in range(4):
        st.ids.copy_(ids)
        offs = st.offsets.clone()
        got = st.step().clone()
        parts = [torch.empty_like(st.logits) for _ in range(world)]
        dist.all_gather(parts, st.logits.contiguous())
        full = torch.cat(parts, dim=1)
        want = ops.sample(full, st.temperature, st.top_k, st.top_p, st.seeds, offs)
        if logprobs:
            lp = ops.logprobs(full, logprobs, tok_ids=want)
            ok = ok and torch.equal(st.top_ids, lp[2])
        torch.cuda.synchronize()
        if not (torch.equal(got, want) and torch.equal(st.offsets, offs)):
            ok = False
            msgs.append((it, got.tolist(), want.tolist(), st.offsets.tolist(), offs.tolist()))
        ids = got
    if st.comm is not None:
        st.comm.check_error()
    extra = {"nccl": 5, "b2": 9, "fused": 9}[collective] + (4 if logprobs else 0) * (collective != "nccl") + \
        (2 if logprobs else 0) * (collective == "nccl")
    recorded = []  # (kernel nodes of a captured step, launches_per_step), sampled and greedy
    if collective == "b2":  # every exchange is a library kernel, so the graph holds exactly the counted launches
        sys.path.insert(0, os.path.join(root, "tests"))
        from test_stack_launches_gpu import graph_kernels, recorded_step
        recorded = [(len(graph_kernels(recorded_step(s))), s.launches_per_step) for s in (st, greedy)]
    ret[rank] = (ok, msgs, st.launches_per_step, greedy.launches_per_step, extra, recorded)
    dist.barrier()
    os._exit(0)  # graphs hold captured collectives: leave without tearing the communicators down


@pytest.mark.parametrize("collective", ["b2", "nccl"])
@pytest.mark.parametrize("logprobs,penalties", [(0, False), (10, True)])
@pytest.mark.parametrize("graph", [False, True])
def test_tp2_sample_matches_whole_row_draw(collective, logprobs, penalties, graph):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, ret, collective, logprobs, penalties, graph)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    for r in range(2):
        ok, msgs, n_sample, n_greedy, extra, recorded = ret[r]
        assert ok, msgs
        assert n_sample == n_greedy + extra, (n_sample, n_greedy, extra)
        assert all(nodes == n for nodes, n in recorded), recorded
