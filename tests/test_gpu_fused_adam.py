"""Target-table Adam folded into the dY epilogue (c2v_arm_target_adam, option "fuse_target_adam").
The epilogue applies the same correctly rounded fp32 operations as adam_kernel to the same
accumulator values, so the target table and its two slots must come out BIT-identical to the
unfused train_step + adam_step pair (tensorflow_model.py:232), with every cta_pair setting, with ragged
tile tails, over several steps, together with lazy Adam and through the host entry point."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

SHAPES = [
    (O.Dims(token_vocab=4001, path_vocab=2003, target_vocab=301, embed_dim=32, code_dim=96, max_contexts=10), 8),
    (O.Dims(token_vocab=999, path_vocab=777, target_vocab=1537, embed_dim=20, code_dim=52, max_contexts=13), 12),
    (O.Dims(token_vocab=5000, path_vocab=3000, target_vocab=2600, embed_dim=128, code_dim=384, max_contexts=16), 64),
]
STEPS = 3


@pytest.mark.parametrize("dims,B", SHAPES)
@pytest.mark.parametrize("cta_pair", [0, 1])
def test_fused_target_adam_is_bit_identical(dims, B, cta_pair):
    import torch
    fused, params0 = make_engine(dims, max_batch=B)
    plain, _ = make_engine(dims, max_batch=B, params=params0)
    for eng in (fused, plain):
        eng.set_option("math_mode", 1)
        eng.set_option("cta_pair", cta_pair)
    for s in range(STEPS):
        src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=300 + s)
        t = s + 1
        fused.arm_target_adam(t)
        for eng in (fused, plain):
            d = dev_batch(eng, src, pth, tgt, mask, target)
            eng.train_step(*d, keep=0.75, seed=5, step=t)
        assert fused.get_option("target_adam_fused_step") == t
        assert plain.get_option("target_adam_fused_step") == 0
        for eng in (fused, plain):
            eng.adam_step(t=t)
        assert fused.get_option("target_adam_fused_step") == 0
    torch.cuda.synchronize()
    for name, a, b in (("theta", fused.params["tgt"], plain.params["tgt"]), ("m", fused.adam_m["tgt"], plain.adam_m["tgt"]),
                       ("v", fused.adam_v["tgt"], plain.adam_v["tgt"])):
        assert torch.equal(a, b), name
    assert not torch.equal(fused.params["tgt"].cpu(), torch.from_numpy(params0["tgt"]))     # it did move
    # the other four tensors took the ordinary path in both engines (embedding scatter order is free)
    a, b = fused.export_params(), plain.export_params()
    for k in ("W", "a"):
        assert np.abs(a[k] - b[k]).max() < 1e-6, k


def test_arming_is_dropped_when_the_step_cannot_fuse_and_mismatches_are_errors():
    import torch
    from code2vec_b200.engine import EngineError
    dims, B = SHAPES[0]
    eng, params0 = make_engine(dims, max_batch=B)
    ref, _ = make_engine(dims, max_batch=B, params=params0)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=1)
    # fp32 SIMT path: no epilogue to fold the update into -> plain dense update, same result as unarmed
    eng.arm_target_adam(1)
    for e in (eng, ref):
        e.train_step(*dev_batch(e, src, pth, tgt, mask, target), keep=1.0)
    assert eng.get_option("target_adam_fused_step") == 0
    for e in (eng, ref):
        e.adam_step(t=1)
    assert torch.equal(eng.params["tgt"], ref.params["tgt"])
    # tf32 path: a fused update must be acknowledged by the matching adam_step
    eng.set_option("math_mode", 1)
    eng.arm_target_adam(2)
    eng.train_step(*dev_batch(eng, src, pth, tgt, mask, target), keep=1.0)
    with pytest.raises(EngineError):
        eng.arm_target_adam(3)                       # previous fused update not acknowledged yet
    with pytest.raises(EngineError):
        eng.adam_step(t=2, lr=5e-3)                  # different hyper-parameters than the armed ones
    eng.adam_t = 1
    eng.adam_step(t=2)                               # the matching call skips the target table


def test_fused_target_adam_with_lazy_adam_through_the_host_entry_point():
    dims, B = SHAPES[0]
    eng, params0 = make_engine(dims, max_batch=B)
    ref, _ = make_engine(dims, max_batch=B, params=params0)
    for e in (eng, ref):
        e.set_option("math_mode", 1)
    eng.set_option("lazy_adam", 1)
    eng.set_option("fuse_target_adam", 1)
    for s in range(5):
        src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=40 + s)
        la = eng.train_batch_host(src, pth, tgt, mask, target, keep=1.0)
        lb = ref.train_batch_host(src, pth, tgt, mask, target, keep=1.0)
        assert abs(la - lb) < 1e-5
    a, b = eng.export_params(), ref.export_params()
    assert np.array_equal(a["tgt"], b["tgt"])
    for k in O.PARAM_NAMES:
        assert np.abs(a[k] - b[k]).max() < 2e-6, k
