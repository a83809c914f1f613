"""Edges of the fused encoder FFN's work split (sdetr_ffn_fused_layernorm): panels of 64 rows, hidden chunks of 128 spread
over the CTAs in contiguous ranges, panels shared by several CTAs finished by a second launch."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F = torch.nn.functional


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


def shared_panels(M, hidden, ctas, sms):
    """Panels whose chunks go to more than one CTA, under the launch's own sizing rule (grid capped at `ctas` or one CTA
    per SM, at the number of units and, with several chunks per panel, at what the workspace holds)."""
    chunks, panels = hidden // 128, (M + 63) // 64
    units = panels * chunks
    g = min(ctas or sms, units)
    if chunks > 1:
        g = min(g, max(1, M * (hidden + 256) // (2 * 64 * 256)))
    starts = [units * i // g for i in range(g)]
    return {u // chunks for u in starts if u % chunks}


def test_ffn_fused_edges(pkg):
    """M = 1, 63, 64, 65, 129 at hidden 128, 256 and 2048, with and without linear2's bias, under the full grid and caps of
    2, 3 and 1 CTAs: against the fp64 reference with the tolerances of test_ffn_fused_layernorm, bit-reproducible, in place;
    shared panels do occur; on one CTA the bare FFN equals the two-GEMM path bit for bit."""
    g = torch.Generator().manual_seed(23)
    lib = pkg.cabi.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    seen_shared = set()
    try:
        for hidden in (128, 256, 2048):
            w1 = (torch.randn(hidden, 256, generator=g) / 16).to(DEV)
            b1 = torch.randn(hidden, generator=g).to(DEV)
            w2 = (torch.randn(256, hidden, generator=g) / hidden ** 0.5).to(DEV)
            b2 = torch.randn(256, generator=g).to(DEV)
            gamma = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV)
            beta = (0.1 * torch.randn(256, generator=g)).to(DEV)
            s1, s2 = pkg.cabi.split_f16_pair(w1), pkg.cabi.split_f16_pair(w2)
            for rows in (1, 63, 64, 65, 129):
                x = torch.randn(rows, 256, generator=g).to(DEV)
                h64 = F.relu(F.linear(x.double(), w1.double(), b1.double()))
                for bias in (b2, None):  # linear2's bias is optional
                    f64 = F.linear(h64, w2.double(), None if bias is None else bias.double())
                    ref = F.layer_norm(x.double() + f64, (256,), gamma.double(), beta.double(), 1e-5)
                    two = pkg.cabi.gemm_f16x3_pre(pkg.cabi.gemm_f16x3_pre(x, *s1, b1, 0), *s2, bias, 1)
                    e_two = (two.double() - f64).abs().max().item()
                    for ctas in (0, 2, 3, 1):
                        lib.sdetr_set_persistent_ctas(ctas)
                        if shared_panels(rows, hidden, ctas, sms):
                            seen_shared.add(hidden)
                        bare = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias)
                        err = (bare.double() - f64).abs().max().item()
                        assert err < 1e-4 and err < 4 * e_two + 1e-6, (rows, hidden, ctas, err, e_two)
                        if ctas == 1:  # every panel on one CTA: the arithmetic of the two-GEMM path, bit for bit
                            assert torch.equal(bare, two), (rows, hidden, bias is None)
                        y = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias, gamma, beta, 1e-5)
                        assert (y.double() - ref).abs().max().item() < 1e-4, (rows, hidden, ctas)
                        assert torch.equal(pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias, gamma, beta, 1e-5), y)
                        xin = x.clone()
                        pkg.cabi.ffn_fused_layernorm(xin, s1, b1, s2, bias, gamma, beta, 1e-5, out=xin)
                        assert torch.equal(xin, y), (rows, hidden, ctas)
    finally:
        lib.sdetr_set_persistent_ctas(0)
    assert seen_shared == {256, 2048}, seen_shared  # one chunk per panel (hidden 128) never shares a panel
