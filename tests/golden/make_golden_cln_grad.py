"""Mints tests/golden/tiny_cln_grad.pt: loss, permutation and every gradient tensor of ``loss.backward()`` through the UNMODIFIED
reference's causal (cLN) Conv-TasNet and PIT1d(NegSISDR), in the reference's fp32 and from the same modules in fp64, on the CPU
(the reference's cLN builds its frame counter there, so the CPU is the only place its causal model runs).  Same record layout as
make_golden.grad_case, every element kept (stride 1).  Run from this directory's make_golden environment:
    python tests/golden/make_golden_cln_grad.py"""
import make_golden as MG

CFG = dict(n_basis=16, kernel_size=4, sep_hidden_channels=16, sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=2,
           sep_num_layers=3, causal=True, n_sources=2)

if __name__ == "__main__":
    MG.grad_case("tiny_cln_grad", MG.O.OracleConfig(**CFG), batch=2, T=203, wseed=12, xseed=22, stride=1)
