"""CPU-side checks of the pure layout / planning logic that the GPU paths rely on (no kernels involved)."""

import pytest
import torch

from torchft_b200.models.llama import CONFIGS, FlatParams, Llama
from torchft_b200.parallel.symm_mem import SymmetricComm


def _flat(cfg_name="llama3_tiny"):
    model = Llama(CONFIGS[cfg_name], device="cpu", dtype=torch.bfloat16)
    return model, FlatParams(model)


def test_flat_params_layout_is_reverse_registration_and_aligned():
    model, flat = _flat()
    names = [n for n, _ in model.named_parameters()]
    assert len(flat.params) == len(names)
    # reverse forward order: the LM head (first gradient of backward) sits at offset 0, the embedding last
    assert flat.params[0] is model.output and flat.params[1] is model.norm and flat.params[-1] is model.tok_embeddings
    assert flat.params[2] is model.layers[-1].w2  # then the last block, last-used parameter first
    assert all(o % FlatParams.ALIGN == 0 for o in flat.offsets)
    assert flat.offsets == sorted(flat.offsets) and flat.numel % FlatParams.ALIGN == 0
    for p, o in zip(flat.params, flat.offsets):
        assert p.data_ptr() == flat.param.data_ptr() + 2 * o  # parameters ARE views of the flat buffer
        assert p._flat_grad.data_ptr() == flat.grad.data_ptr() + 2 * o and p._flat_grad.shape == p.shape


def test_flat_params_buckets_tile_the_buffer_in_backward_order():
    _, flat = _flat()
    for bucket_elems in (1, 5000, 10 ** 9):
        buckets = flat.buckets(bucket_elems)
        assert buckets[0][0] == 0 and buckets[-1][1] == flat.numel
        assert all(a[1] == b[0] for a, b in zip(buckets, buckets[1:]))
        assert sum(len(b[2]) for b in buckets) == len(flat.params)
        if bucket_elems == 10 ** 9:
            assert len(buckets) == 1
    # reset_grads(zero=False) drops p.grad so producers write the flat buffer directly; adopt_grad re-homes one
    flat.reset_grads()
    assert all(p.grad is None for p in flat.params)
    p = flat.params[3]
    p.grad = torch.ones_like(p)
    flat.adopt_grad(p)
    assert p.grad.data_ptr() == p._flat_grad.data_ptr() and bool((p._flat_grad == 1).all())
    flat.reset_grads(zero=True)
    assert all(pp.grad is pp._flat_grad for pp in flat.params) and float(flat.grad.abs().sum()) == 0.0


def test_param_stages_tile_the_flat_buffer_in_forward_order():
    """The per-stage AdamW of the trainer relies on this: stages = [embedding], blocks..., [norm, head]."""
    model, flat = _flat("llama3_debug")
    where = {id(p): (o, p.numel()) for p, o in zip(flat.params, flat.offsets)}
    stages = model.param_stages()
    assert len(stages) == model.cfg.n_layers + 2
    ranges = []
    for st in stages:
        lo = min(where[id(p)][0] for p in st)
        hi = max((where[id(p)][0] + where[id(p)][1] + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN for p in st)
        ranges.append((lo, min(hi, flat.numel)))
    # forward order runs from the END of the flat buffer to its start, without gaps or overlap
    assert ranges[0][1] == flat.numel and ranges[-1][0] == 0
    assert all(a[0] == b[1] for a, b in zip(ranges, ranges[1:]))
    # and the buckets of the gradient all-reduce start with the head (first gradients of backward)
    first_bucket = flat.buckets(1)[0]
    assert first_bucket[2][0] is model.output
    assert {id(p) for st in stages for p in st} == {id(p) for p in flat.params}


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_allreduce_plan_is_well_formed(world):
    comm = SymmetricComm.__new__(SymmetricComm)  # planning needs no device state
    comm._force_plan, comm._world, comm._oneshot_max, comm._max_blocks = None, world, 256 << 10, 64
    prev_algo = 0
    for k in range(4, 31):
        nbytes = 1 << k
        algo, blocks = SymmetricComm._plan(comm, nbytes)
        assert algo in (0, 1) and 1 <= blocks <= 128
        if algo == 0:  # one-shot keeps results in registers across the closing barrier: <= 64 KB per CTA
            assert (nbytes + blocks - 1) // blocks <= (64 << 10)
        else:
            assert 8 <= blocks <= comm._max_blocks
        assert algo >= prev_algo, "once two-shot wins it keeps winning for larger messages"
        prev_algo = algo
    # the plan's cross-overs: two-shot from 256 KB at 8 replicas, one-shot up to 2 MB at 2
    assert SymmetricComm._plan(comm, 4 << 20)[0] == 1
    assert SymmetricComm._plan(comm, 64 << 10)[0] == 0
    assert SymmetricComm._default_nvls_min(2) > (1 << 40) and SymmetricComm._default_nvls_min(4) > (1 << 40)
    assert SymmetricComm._default_nvls_min(8) == 256 << 10
