"""sige_sparse_attention at head dim 512 — the single head of the Stable Diffusion VAE's mid-block attention — against the float64
restatement of its contract (tests/step_kernel_contracts.py): the per-element bound on every element written, every other element
(guard bands included) and every input bitwise unchanged, a repeat bitwise equal.  Query counts around the CTA's 64 rows and the
~800 active tokens of a 15 % edit of a 64 x 64 latent; key counts from one to 9216, so that the key range is split over clusters
of 1 to 8 CTAs.  The worst error / bound ratio of each launch is printed (pytest -s)."""
import pytest
import torch

import step_kernel_contracts as sk
from kernel_contracts import _run_and_check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
P = sk.SAttnSpec
CASES = [
    P("q1_k1", 1, 1, 1, 1, 512, seed=1),
    P("q63_k65_bnhd", 1, 1, 63, 65, 512, layout="bnhd", seed=2),
    P("q64_k4096", 1, 1, 64, 4096, 512, seed=3),
    P("q65_k9216_bnhd", 1, 1, 65, 9216, 512, layout="bnhd", seed=4),
    P("q800_k4096", 1, 1, 800, 4096, 512, seed=5),
    P("q800_k9216_bnhd", 1, 1, 800, 9216, 512, layout="bnhd", seed=6),
    P("q64_k1_bnhd", 1, 1, 64, 1, 512, layout="bnhd", seed=7),
    P("q65_k65", 1, 1, 65, 65, 512, seed=8),
    P("q1_k4096_bnhd", 1, 1, 1, 4096, 512, layout="bnhd", seed=9),
    P("q63_k9216_falling", 1, 1, 63, 9216, 512, mode="falling", seed=10),
    P("q65_k4096_dominant_last_bnhd", 1, 1, 65, 4096, 512, mode="dominant", dom="last", layout="bnhd", seed=11),
    P("q800_k65_dominant_first", 1, 1, 800, 65, 512, mode="dominant", seed=12),
    P("q64_k4096_constant_v", 1, 1, 64, 4096, 512, mode="constant_v", seed=13),
    P("b2_q65_k130_bnhd", 2, 1, 65, 130, 512, layout="bnhd", seed=14),
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", CASES, ids=lambda s: s.name)
def test_wide_head_sparse_attention_matches_the_float64_contract(spec, dtype):
    from sige_b200 import _cabi

    lib = _cabi.lib()
    assert lib.sige_sparse_attention_supported(512, sk._code(dtype)) == 1
    case = sk.make_sattn(spec, dtype, DEV)
    expects = sk.sattn_reference(case, chunk=4)
    d = sk.sattn_descriptor(case)
    _run_and_check("sparse_att_d512", "%s %s" % (spec.name, "f16" if dtype == torch.float16 else "bf16"), case, expects,
                   lambda flags: sk.sattn_call(case, lib, d))


def test_wide_head_with_no_queries_is_a_no_op():
    from sige_b200 import ops

    q = torch.empty(1, 0, 512, dtype=torch.float16, device=DEV)
    k = torch.randn(1, 70, 512, dtype=torch.float16, device=DEV)
    out = torch.empty(1, 0, 512, dtype=torch.float16, device=DEV)
    ops.sparse_attention(q, k, k, 512 ** -0.5, out=out)
    torch.cuda.synchronize()
