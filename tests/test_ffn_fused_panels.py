"""Edges of the fused encoder FFN's 128-row panels (sdetr_ffn_fused_layernorm): two consumer warpgroups of 64 rows each,
hidden chunks of 64 spread over the CTAs in contiguous ranges, panels shared by several CTAs finished by a second launch."""
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
    """Panels of 128 rows whose 64-wide hidden chunks go to more than one CTA, under the launch's sizing rule (grid capped
    at `ctas` or one CTA per SM, at the number of units and at the two 128 x 256 partial slots per CTA that the workspace
    of M * (hidden + 256) floats holds)."""
    chunks, panels = hidden // 64, (M + 127) // 128
    units = panels * chunks
    g = min(ctas or sms, units)
    g = min(g, max(1, M * (hidden + 256) // (2 * 128 * 256)))
    starts = [units * i // g for i in range(g)]
    return {u // chunks for u in starts if u % chunks}


def test_ffn_fused_panel_edges(pkg):
    """M around the 64-row warpgroup halves and the 128-row panels (and 383, where hidden 128 shares a panel), at hidden
    128, 256 and 2048, with and without linear2's bias, under the full grid and caps of 1, 2 and 3 CTAs: against the fp64
    reference, bit-reproducible, in place; shared panels do occur; on one CTA the bare FFN equals the two-GEMM path bit
    for bit."""
    g = torch.Generator().manual_seed(29)
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
            for rows in (1, 63, 64, 65, 127, 128, 129, 255, 257, 383):
                x = torch.randn(rows, 256, generator=g).to(DEV)
                h64 = F.relu(F.linear(x.double(), w1.double(), b1.double()))
                for bias in (b2, None):
                    f64 = F.linear(h64, w2.double(), None if bias is None else bias.double())
                    ref = F.layer_norm(x.double() + f64, (256,), gamma.double(), beta.double(), 1e-5)
                    two = pkg.cabi.gemm_f16x3_pre(pkg.cabi.gemm_f16x3_pre(x, *s1, b1, 0), *s2, bias, 1)
                    e_two = (two.double() - f64).abs().max().item()
                    for ctas in (0, 1, 2, 3):
                        lib.sdetr_set_persistent_ctas(ctas)
                        if shared_panels(rows, hidden, ctas, sms):
                            seen_shared.add(hidden)
                        bare = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias)
                        err = (bare.double() - f64).abs().max().item()
                        assert err < 1e-4 and err < 4 * e_two + 1e-6, (rows, hidden, ctas, err, e_two)
                        if ctas == 1:
                            assert torch.equal(bare, two), (rows, hidden, bias is None)
                        y = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias, gamma, beta, 1e-5)
                        assert (y.double() - ref).abs().max().item() < 1e-4, (rows, hidden, ctas)
                        assert torch.equal(pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, bias, gamma, beta, 1e-5), y)
                        xin = x.clone()
                        pkg.cabi.ffn_fused_layernorm(xin, s1, b1, s2, bias, gamma, beta, 1e-5, out=xin)
                        assert torch.equal(xin, y), (rows, hidden, ctas)
    finally:
        lib.sdetr_set_persistent_ctas(0)
    assert seen_shared == {128, 256, 2048}, seen_shared  # 64-wide chunks: even hidden 128 has two per panel (M = 383)
