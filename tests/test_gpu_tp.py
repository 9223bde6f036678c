"""2-GPU check of the column -> row sharded MLP with the NCCL all-reduce (skipped with fewer than 2 GPUs).
Compares the tensor-parallel result on this repository's kernels with the unsharded oracle contraction."""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import awq_oracle as O

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from autoawq_b200 import shard as S

        K, I, G = 1024, 2048, 128
        dev = torch.device("cuda", rank)

        def packed(c):
            return S.PackedGemm(torch.from_numpy(c["qweight"]).to(dev), torch.from_numpy(c["qzeros"]).to(dev),
                                torch.from_numpy(c["scales"]).to(dev))

        cg, cu, cd = O.make_case(K, I, G, seed=1), O.make_case(K, I, G, seed=2), O.make_case(I, K, G, seed=3)
        mlp = S.TensorParallelMLP(packed(cg), packed(cu), packed(cd), rank, world)
        for M in (1, 24):
            x = (np.random.default_rng(M).standard_normal((M, K)) * 0.5).astype(np.float16)
            y = mlp(torch.from_numpy(x).to(dev)).float().cpu().numpy()
            wg = O.dequantize_gemm(cg["qweight"], cg["qzeros"], cg["scales"], G)
            wu = O.dequantize_gemm(cu["qweight"], cu["qzeros"], cu["scales"], G)
            wd = O.dequantize_gemm(cd["qweight"], cd["qzeros"], cd["scales"], G)
            g = O.gemm_f64(x, wg).astype(np.float16).astype(np.float64)
            u = O.gemm_f64(x, wu).astype(np.float16).astype(np.float64)
            act = (g / (1 + np.exp(-g)) * u).astype(np.float16)
            ref = O.gemm_f64(act, wd)
            # two fp16 roundings upstream + fp16 partial sums reduced across ranks
            tol = 4e-3 * np.abs(ref) + 2e-3 * np.sqrt(np.mean(ref**2)) + 1e-4
            assert np.all(np.abs(y - ref) <= tol), f"rank {rank} M={M}: max err {np.abs(y - ref).max()}"
        # ---- the one-shot all-reduce over peer memory (csrc/comm.cu) against the sum of the gathered partials
        from autoawq_b200.comm import OneShotAllReduce

        ar = OneShotAllReduce(max_elems=8192)
        g = torch.Generator(device=dev).manual_seed(100 + rank)
        for it, n in enumerate([8192, 4096, 8, 8192, 8192]):       # several calls: both parities, reuse
            part = torch.randn(n, device=dev, dtype=torch.float16, generator=g)
            parts = [torch.empty_like(part) for _ in range(world)]
            dist.all_gather(parts, part)
            want = sum(p.float() for p in parts).half()            # rank order, fp32 accumulation, one rounding
            got = ar(part.clone())
            torch.cuda.synchronize()
            assert torch.equal(got, want), f"rank {rank} call {it}: one-shot all-reduce differs from the rank-ordered sum"
        # inside a CUDA graph, replayed: the call counter lives on the device
        buf = torch.zeros(8192, device=dev, dtype=torch.float16)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ar(buf)
            s.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=s):
                ar(buf)
            for rep in range(5):
                buf.fill_(float(rank + 1 + rep))
                gr.replay()
                s.synchronize()
                assert float(buf[0]) == sum(r + 1 + rep for r in range(world)), f"rank {rank} replay {rep}"
        ar.check()
        # the tensor-parallel MLP with the one-shot collective gives the same result as with NCCL (same partials;
        # NCCL's reduction order may differ in the last bit)
        mlp1 = S.TensorParallelMLP(packed(cg), packed(cu), packed(cd), rank, world, all_reduce=ar)
        x = torch.from_numpy((np.random.default_rng(5).standard_normal((1, K)) * 0.5).astype(np.float16)).to(dev)
        ya, yb = mlp1(x).float(), mlp(x).float()
        assert torch.allclose(ya, yb, rtol=2e-3, atol=2e-3)
        ret[rank] = True
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tensor_parallel_mlp_nccl():
    import torch.multiprocessing as mp

    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
        assert ret.get(0) and ret.get(1)
