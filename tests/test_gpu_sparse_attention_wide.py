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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("spec", sk.WIDE_CASES, ids=lambda s: s.name)
def test_wide_head_sparse_attention_matches_the_float64_contract(spec, dtype):
    """Within the bound of the wide kernel's own algorithm (sk.wide_sattn_reference); the worst ratio under the bound of the
    64-key single-range kernel (sk.sattn_reference) is printed beside it."""
    from sige_b200 import _cabi

    lib = _cabi.lib()
    assert lib.sige_sparse_attention_supported(512, sk._code(dtype)) == 1
    case = sk.make_sattn(spec, dtype, DEV)
    expects = sk.wide_sattn_reference(case, _sms(), chunk=4)
    d = sk.sattn_descriptor(case)
    label = "%s %s cs=%d" % (spec.name, "f16" if dtype == torch.float16 else "bf16", sk.wide_cluster(spec.Nq, spec.Nk, spec.B * spec.heads, _sms()))
    got = _run_and_check("sparse_att_d512", label, case, expects, lambda flags: sk.sattn_call(case, lib, d))
    (old,) = sk.sattn_reference(case, chunk=4)
    w = old.written
    err = (got["out"].double()[w] - old.want[w]).abs()
    print("[kernel contract] sparse_att_d512 %-52s worst |err| / old bound %.3f" % (label, float((err / old.bound[w]).max())))


def test_wide_head_with_no_queries_is_a_no_op():
    from sige_b200 import ops

    q = torch.empty(1, 0, 512, dtype=torch.float16, device=DEV)
    k = torch.randn(1, 70, 512, dtype=torch.float16, device=DEV)
    out = torch.empty(1, 0, 512, dtype=torch.float16, device=DEV)
    ops.sparse_attention(q, k, k, 512 ** -0.5, out=out)
    torch.cuda.synchronize()
