"""GPU parity of the attention / normalisation / elementwise kernels against fp32 torch math."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
DEV = "cuda:0"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _close(got, ref, tol=2e-2, what=""):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    rel = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    mx = (got - ref).abs().max().item()
    assert rel < tol and mx < 8 * tol * max(ref.abs().max().item(), 1e-6), (
        f"{what}: rel-l2 {rel:.4g} max-abs {mx:.4g} (ref max {ref.abs().max().item():.4g})")


@pytest.fixture(scope="module")
def raw():
    from svd_xtend_b200 import raw
    return raw


def _sdpa_ref(q, k, v, scale):
    # q,k,v: [nseq, S, heads, 64] fp32
    qh, kh, vh = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    att = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (att @ vh).permute(0, 2, 1, 3)


@pytest.mark.parametrize("nseq,S,heads", [(2, 256, 2), (3, 640, 5), (2, 160, 3), (4, 40, 2), (1, 2560, 1), (1, 9216, 1), (2, 2304, 2), (3, 144, 2)])
def test_attention_spatial_fwd_bwd(raw, nseq, S, heads):
    C = heads * 64
    qkv = _rand(nseq * S, 3 * C, seed=1).to(bf16)          # fused projection buffer: q|k|v column slices
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    o = torch.zeros(nseq * S, C, device=DEV, dtype=bf16)
    lse = torch.zeros(nseq * S, heads, device=DEV)
    raw.attention_fwd(q, k, v, o, heads=heads, S=S, nseq=nseq, lse=lse)
    torch.cuda.synchronize()
    qf, kf, vf = (t.float().reshape(nseq, S, heads, 64).requires_grad_(True) for t in (q, k, v))
    ref = _sdpa_ref(qf, kf, vf, 0.125)
    _close(o.view(nseq, S, heads, 64), ref, what="attn fwd")
    sc = torch.einsum("nqhd,nkhd->nhqk", qf, kf) * 0.125
    _close(lse.view(nseq, S, heads), torch.logsumexp(sc, -1).permute(0, 2, 1), tol=2e-3, what="lse")
    dout = _rand(nseq * S, C, seed=2).to(bf16)
    dqkv = torch.zeros_like(qkv)
    delta = torch.zeros_like(lse)
    raw.attention_bwd(q, k, v, o, dout, dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:], lse, delta, heads=heads, S=S, nseq=nseq)
    torch.cuda.synchronize()
    ref.backward(dout.float().view(nseq, S, heads, 64))
    _close(dqkv[:, :C].reshape(nseq, S, heads, 64), qf.grad, tol=3e-2, what="dq")
    _close(dqkv[:, C:2 * C].reshape(nseq, S, heads, 64), kf.grad, tol=3e-2, what="dk")
    _close(dqkv[:, 2 * C:].reshape(nseq, S, heads, 64), vf.grad, tol=3e-2, what="dv")


@pytest.mark.parametrize("B,T,HW,heads", [(1, 14, 160, 2), (2, 14, 40, 3), (1, 25, 144, 2), (1, 4, 64, 1)])
def test_attention_temporal_fwd_bwd(raw, B, T, HW, heads):
    # tokens are [B, T, HW] row-major; a sequence = fixed (b, pixel), tokens strided by HW
    C = heads * 64
    M = B * T * HW
    qkv = _rand(M, 3 * C, seed=3).to(bf16)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    o = torch.zeros(M, C, device=DEV, dtype=bf16)
    lse = torch.zeros(M, heads, device=DEV)
    geo = dict(heads=heads, S=T, nseq=B * HW, inner=HW, outer_stride=T * HW, inner_stride=1, tok_stride=HW)
    raw.attention_fwd(q, k, v, o, lse=lse, **geo)
    torch.cuda.synchronize()

    def to_seq(t):  # [M, C] -> [B*HW, T, heads, 64]
        return t.float().reshape(B, T, HW, heads, 64).permute(0, 2, 1, 3, 4).reshape(B * HW, T, heads, 64)

    qf, kf, vf = (to_seq(t).requires_grad_(True) for t in (q, k, v))
    ref = _sdpa_ref(qf, kf, vf, 0.125)
    _close(to_seq(o), ref, what="temporal attn fwd")
    dout = _rand(M, C, seed=4).to(bf16)
    dqkv = torch.zeros_like(qkv)
    delta = torch.zeros_like(lse)
    raw.attention_bwd(q, k, v, o, dout, dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:], lse, delta, **geo)
    torch.cuda.synchronize()
    ref.backward(to_seq(dout))
    _close(to_seq(dqkv[:, :C]), qf.grad, tol=3e-2, what="temporal dq")
    _close(to_seq(dqkv[:, C:2 * C]), kf.grad, tol=3e-2, what="temporal dk")
    _close(to_seq(dqkv[:, 2 * C:]), vf.grad, tol=3e-2, what="temporal dv")


@pytest.mark.parametrize("outer,rows,C1,C2,silu", [(14, 160, 320, 0, True), (3, 640, 1280, 640, True), (2, 14 * 40, 640, 0, False), (2, 100, 640, 320, True),
                                                  (1, 35841, 320, 0, True), (2, 9001, 320, 320, False)])   # long slabs: the cp.async rings wrap
def test_groupnorm_fwd_bwd_through_channel_sums(raw, outer, rows, C1, C2, silu):
    """the stand-alone channel-sum kernels (one or two sources) feeding the same consumers as the epilogue sums"""
    C = C1 + C2
    x1 = _rand(outer * rows, C1, seed=5).to(bf16) + 0.5
    x2 = _rand(outer * rows, C2, seed=6).to(bf16) if C2 else None
    gamma = _rand(C, seed=7) * 0.2 + 1.0
    beta = _rand(C, seed=8) * 0.1
    sums = raw.groupnorm_sums(x1, x2, outer, rows)
    y = torch.empty(outer * rows, C, device=DEV, dtype=bf16)
    ab = torch.empty(outer, 2, C, device=DEV)
    mean, rstd = raw.groupnorm_apply_fused(x1, x2, outer, rows, 1e-5, sums, sums[:, :, C1:] if C2 else None, gamma, beta, silu, y, ab=ab)
    torch.cuda.synchronize()
    xcat = torch.cat([x1, x2], 1) if C2 else x1
    xr = xcat.float().reshape(outer, rows, C).permute(0, 2, 1).requires_grad_(True)  # [outer, C, rows]
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    ref = F.group_norm(xr, 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    _close(y.view(outer, rows, C), ref.permute(0, 2, 1), what="groupnorm fwd")
    dy = _rand(outer * rows, C, seed=9).to(bf16)
    dx1 = torch.zeros_like(x1)
    dx2 = torch.zeros_like(x2) if C2 else None
    dgamma = torch.zeros(C, device=DEV)
    dbeta = torch.zeros(C, device=DEV)
    bsums = raw.groupnorm_bwd_sums(x1, x2, dy, outer, rows, ab, silu)
    raw.groupnorm_bwd_fused(x1, x2, dy, outer, rows, mean, rstd, gamma, beta, silu, bsums, dx1, dx2, dgamma, dbeta)
    torch.cuda.synchronize()
    ref.backward(dy.float().view(outer, rows, C).permute(0, 2, 1))
    dxr = xr.grad.permute(0, 2, 1).reshape(outer * rows, C)
    _close(dx1, dxr[:, :C1], what="groupnorm dx")
    if C2:
        _close(dx2, dxr[:, C1:], what="groupnorm dx2")
    _close(dgamma, g.grad, what="groupnorm dgamma")
    _close(dbeta, b.grad, what="groupnorm dbeta")
    if not C2:      # residual gradient folded into the same pass (single-source form)
        dres = _rand(outer * rows, C, seed=10).to(bf16)
        dx3 = torch.zeros_like(x1)
        raw.groupnorm_bwd_fused(x1, None, dy, outer, rows, mean, rstd, gamma, beta, silu, bsums, dx3, None, dres=dres)
        torch.cuda.synchronize()
        _close(dx3, dxr + dres.float(), what="groupnorm dx + dres")


@pytest.mark.parametrize("rows,C", [(1000, 320), (560, 1280), (77, 64), (300, 640), (40003, 320), (30001, 640), (20011, 1280), (1500, 960), (130, 2048)])   # C > 1280: the register-array kernels
def test_layernorm_fwd_bwd(raw, rows, C):
    x = (_rand(rows, C, seed=10) + 0.3).to(bf16)
    gamma = _rand(C, seed=11) * 0.2 + 1.0
    beta = _rand(C, seed=12) * 0.1
    y = torch.empty_like(x)
    mean, rstd = raw.layernorm_fwd(x, gamma, beta, 1e-5, y)
    torch.cuda.synchronize()
    xr = x.float().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    ref = F.layer_norm(xr, (C,), g, b, 1e-5)
    _close(y, ref, what="layernorm fwd")
    dy = _rand(rows, C, seed=13).to(bf16)
    dres = _rand(rows, C, seed=14).to(bf16)
    dx = torch.empty_like(x)
    dgamma = torch.zeros(C, device=DEV)
    dbeta = torch.zeros(C, device=DEV)
    raw.layernorm_bwd(x, dy, gamma, mean, rstd, dx, dres, dgamma, dbeta)
    torch.cuda.synchronize()
    ref.backward(dy.float())
    _close(dx, xr.grad + dres.float(), what="layernorm dx")
    _close(dgamma, g.grad, what="layernorm dgamma")
    _close(dbeta, b.grad, what="layernorm dbeta")
    # the other three instantiations: no parameter gradients and / or no residual gradient
    dx2 = torch.empty_like(x)
    raw.layernorm_bwd(x, dy, gamma, mean, rstd, dx2, dres)
    torch.cuda.synchronize()
    _close(dx2, xr.grad + dres.float(), what="layernorm dx (no dgamma)")
    dx3 = torch.empty_like(x)
    raw.layernorm_bwd(x, dy, gamma, mean, rstd, dx3)
    torch.cuda.synchronize()
    _close(dx3, xr.grad, what="layernorm dx (no dres)")
    dx4 = torch.empty_like(x)
    dg4 = torch.zeros(C, device=DEV)
    db4 = torch.zeros(C, device=DEV)
    raw.layernorm_bwd(x, dy, gamma, mean, rstd, dx4, None, dg4, db4)
    torch.cuda.synchronize()
    _close(dx4, xr.grad, what="layernorm dx (dgamma, no dres)")
    _close(dg4, g.grad, what="layernorm dgamma (no dres)")
    # x + addvec (per-frame vector, broadcast over add_div rows) rounded to bf16 is both an output and the normalised value
    div = max(rows // 7, 1)
    nvec = (rows + div - 1) // div
    addvec = _rand(nvec, C, seed=15) * 0.5
    xsum = torch.empty_like(x)
    y2 = torch.empty_like(x)
    raw.layernorm_fwd(x, gamma, beta, 1e-5, y2, addvec=addvec, add_div=div, xsum=xsum)
    torch.cuda.synchronize()
    xs_ref = (x.float() + addvec.repeat_interleave(div, 0)[:rows]).to(bf16)
    assert torch.equal(xsum, xs_ref)
    _close(y2, F.layer_norm(xs_ref.float(), (C,), gamma, beta, 1e-5), what="layernorm fwd (+addvec)")


def test_prep_weight_layouts(raw):
    O, I, T = 96, 40, 9
    w = _rand(O, I, T, seed=15)
    d2 = torch.empty(O, T, 64, device=DEV, dtype=bf16)
    raw.prep_weight(w, d2, 2, O, I, T, 64)
    d3 = torch.empty(I, T, O, device=DEV, dtype=bf16)
    raw.prep_weight(w, d3, 3, O, I, T)
    wl = _rand(O, I, seed=16)
    d0 = torch.empty(O, I, device=DEV, dtype=bf16)
    d1 = torch.empty(I, O, device=DEV, dtype=bf16)
    raw.prep_weight(wl, d0, 0, O, I)
    raw.prep_weight(wl.to(bf16), d1, 1, O, I)
    torch.cuda.synchronize()
    ref2 = torch.zeros(O, T, 64, device=DEV)
    ref2[:, :, :I] = w.permute(0, 2, 1)
    assert torch.equal(d2, ref2.to(bf16))
    assert torch.equal(d3, w.permute(1, 2, 0).contiguous().to(bf16))
    assert torch.equal(d0, wl.to(bf16))
    assert torch.equal(d1, wl.to(bf16).t().contiguous())


def test_layout_kernels(raw):
    N, C, H, W = 3, 8, 10, 16
    x = _rand(N, C, H, W, seed=17)
    nhwc = torch.empty(N, H, W, 64, device=DEV, dtype=bf16)
    raw.nchw_to_nhwc(x, nhwc, N, C, H, W, 64)
    back = torch.empty(N, C, H, W, device=DEV)
    raw.nhwc_to_nchw(nhwc.view(-1, 64), back, N, C, H, W)
    torch.cuda.synchronize()
    assert torch.equal(nhwc[..., :C], x.permute(0, 2, 3, 1).to(bf16)) and (nhwc[..., C:] == 0).all()
    assert torch.equal(back, x.to(bf16).float())
    a = _rand(N, H, W, 64, seed=18).to(bf16)
    up = torch.empty(N, 2 * H, 2 * W, 64, device=DEV, dtype=bf16)
    raw.upsample2x(a, up, N, H, W, 64)
    torch.cuda.synchronize()
    ref = F.interpolate(a.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), ref)
    dup = _rand(N, 2 * H, 2 * W, 64, seed=19).to(bf16)
    da = torch.empty_like(a)
    raw.upsample2x_bwd(dup, da, N, H, W, 64)
    torch.cuda.synchronize()
    refd = dup.float().view(N, H, 2, W, 2, 64).sum((2, 4))
    _close(da, refd, tol=1e-2, what="upsample bwd")
    planes = torch.empty(4 * N, H // 2, W // 2, 64, device=DEV, dtype=bf16)
    raw.space_to_planes(a, planes, N, H, W, 64)
    a2 = torch.empty_like(a)
    raw.planes_to_space(planes, a2, N, H, W, 64)
    torch.cuda.synchronize()
    for p in range(2):
        for q in range(2):
            assert torch.equal(planes[(p * 2 + q) * N:(p * 2 + q + 1) * N], a[:, p::2, q::2])
    assert torch.equal(a2, a)
    b = _rand(N, H, W, 128, seed=20).to(bf16)
    cat = torch.empty(N, H, W, 192, device=DEV, dtype=bf16)
    raw.concat_channels(a, b, cat)
    a3, b3 = torch.empty_like(a), torch.empty_like(b)
    raw.split_channels(cat, a3, b3)
    torch.cuda.synchronize()
    assert torch.equal(cat, torch.cat([a, b], -1)) and torch.equal(a3, a) and torch.equal(b3, b)


def test_misc_elementwise(raw):
    rows, h = 333, 256
    pre = _rand(rows, 2 * h, seed=21).to(bf16)
    dout = _rand(rows, h, seed=22).to(bf16)
    dpre = torch.empty_like(pre)
    raw.geglu_bwd(pre, dout, dpre)
    pr = pre.float().requires_grad_(True)
    (pr[:, :h] * F.gelu(pr[:, h:])).backward(dout.float())
    torch.cuda.synchronize()
    _close(dpre, pr.grad, what="geglu bwd")
    # fused bias gradient of the projection: column sums of the dpre that was written (accumulating), ragged row count
    for rows2, h2 in ((333, 256), (35840, 1280), (17, 64)):
        pre2 = _rand(rows2, 2 * h2, seed=31).to(bf16)
        dout2 = _rand(rows2, h2, seed=32).to(bf16)
        dpre2 = torch.empty_like(pre2)
        bg = torch.full((2 * h2,), 0.5, device=DEV)
        raw.geglu_bwd(pre2, dout2, dpre2, bias_grad=bg)
        torch.cuda.synchronize()
        ref2 = torch.empty_like(pre2)
        raw.geglu_bwd(pre2, dout2, ref2)
        torch.cuda.synchronize()
        assert torch.equal(dpre2, ref2)
        _close(bg, 0.5 + dpre2.float().sum(0), tol=2e-3, what=f"geglu bwd fused bias gradient {rows2}x{h2}")
    x = _rand(5000, 320, seed=23).to(bf16)
    out = torch.empty(320, device=DEV)
    raw.colsum(x, out)
    torch.cuda.synchronize()
    _close(out, x.float().sum(0), tol=1e-3, what="colsum")
    mix = torch.tensor([0.5], device=DEV)
    s3 = torch.empty(16, device=DEV)
    raw.blend_scales(mix, s3)
    a = torch.sigmoid(mix)
    one, zero = torch.ones_like(a), torch.zeros_like(a)
    torch.cuda.synchronize()
    assert torch.allclose(s3, torch.stack([1 - a, a, 1 - a, zero, 1 - a, one, zero, a * (1 - a), 1 - a, zero, zero, zero, a, zero, 1 - a, zero]).flatten(), atol=1e-6)
    y = torch.empty_like(x)
    raw.axpby(x, x, y, s3)
    torch.cuda.synchronize()
    _close(y, x.float() * (s3[0] + s3[1]), tol=1e-2, what="axpby")
    # AdamW vs torch, at a length whose last elements take the kernel's scalar tail
    p0 = _rand(1003, seed=24)
    g = _rand(1003, seed=25)
    p = p0.clone()
    pt = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pt], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
    for step in (1, 2, 3):
        pt.grad = g.clone()
        opt.step()
        raw.adamw_graph(p, g, m, v, state)
    torch.cuda.synchronize()
    assert torch.allclose(p, pt.detach(), atol=1e-5, rtol=1e-5)
    # the tail's bits are the vector body's: the same three elements updated as part of a 4-element buffer
    p4, g4 = torch.cat([p0[1000:], p0[:1]]), torch.cat([g[1000:], g[:1]])
    m4, v4, state4 = torch.zeros_like(p4), torch.zeros_like(p4), torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
    for _ in range(3):
        raw.adamw_graph(p4, g4, m4, v4, state4)
    torch.cuda.synchronize()
    assert torch.equal(p4[:3], p[1000:]) and torch.equal(m4[:3], m[1000:]) and torch.equal(v4[:3], v[1000:])


def test_multi_transpose_bit_exact(raw):
    """All dgrad operand transposes in one launch (train.ParamArena.refresh_transposes): ragged and odd shapes."""
    import struct
    shapes = [(320, 320), (1280, 320), (96, 200), (33, 65), (64, 1), (5, 7), (640, 2560)]
    offs, total = [], 0
    for O, I in shapes:
        offs.append(total)
        total += ((O * I + 63) // 64) * 64
    src = torch.randn(total, device=DEV).to(bf16)
    dsts = [torch.zeros(I, O, device=DEV, dtype=bf16) for O, I in shapes]
    blob, prefix, tiles = bytearray(), [], 0
    for (O, I), off, d in zip(shapes, offs, dsts):
        blob += struct.pack("<qqii", off, d.data_ptr(), O, I)
        prefix.append(tiles)
        tiles += ((O + 63) // 64) * ((I + 63) // 64)
    jobs = torch.frombuffer(bytes(blob), dtype=torch.uint8).clone().to(DEV)
    pre = torch.tensor(prefix, dtype=torch.int32, device=DEV)
    raw.multi_transpose(src, jobs, pre, len(shapes), tiles)
    torch.cuda.synchronize()
    for (O, I), off, d in zip(shapes, offs, dsts):
        ref = src[off:off + O * I].view(O, I).t().contiguous()
        assert torch.equal(d, ref), f"transpose {O}x{I}"


@pytest.mark.parametrize("outer,rows,C1,C2,silu", [(14, 2560, 320, 0, True), (14, 160, 1280, 640, True), (2, 560, 640, 320, False),
                                                    (3, 40, 1280, 1280, True), (1, 1000, 64, 0, True)])
def test_groupnorm_fwd_bwd_from_given_channel_sums(raw, outer, rows, C1, C2, silu):
    """svdx_groupnorm_apply_fused: group statistics folded from per-channel sums (as the GEMM epilogues produce them), one or
    two channel-concatenated sources, against F.group_norm; mean / rstd published for the backward."""
    C = C1 + C2
    x1 = _rand(outer * rows, C1, seed=5).to(bf16) + 0.5
    x2 = _rand(outer * rows, C2, seed=6).to(bf16) if C2 else None
    gamma = _rand(C, seed=7) * 0.2 + 1.0
    beta = _rand(C, seed=8) * 0.1

    def sums(t):
        v = t.float().view(outer, rows, -1)
        return torch.stack([v.sum(1), (v * v).sum(1)], dim=1).contiguous()      # [outer, 2, Ci]

    y = torch.empty(outer * rows, C, device=DEV, dtype=bf16)
    ab = torch.empty(outer, 2, C, device=DEV)
    mean, rstd = raw.groupnorm_apply_fused(x1, x2, outer, rows, 1e-5, sums(x1), sums(x2) if C2 else None, gamma, beta, silu, y, ab=ab)
    torch.cuda.synchronize()
    xcat = torch.cat([x1, x2], 1) if C2 else x1
    xr = xcat.float().reshape(outer, rows, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    _close(y.view(outer, rows, C), ref.permute(0, 2, 1), what="groupnorm fused fwd")
    v = xr.reshape(outer, 32, -1)
    assert torch.allclose(mean.view(outer, 32), v.mean(-1), atol=1e-4, rtol=1e-4)
    assert torch.allclose(rstd.view(outer, 32), torch.rsqrt(v.var(-1, unbiased=False) + 1e-5), atol=1e-3, rtol=1e-3)
    # the published statistics and scale / shift table drive the backward kernels
    dy = _rand(outer * rows, C, seed=9).to(bf16)
    dx1 = torch.zeros_like(x1)
    dx2 = torch.zeros_like(x2) if C2 else None
    bsums = raw.groupnorm_bwd_sums(x1, x2, dy, outer, rows, ab, silu)
    raw.groupnorm_bwd_fused(x1, x2, dy, outer, rows, mean, rstd, gamma, beta, silu, bsums, dx1, dx2)
    torch.cuda.synchronize()
    xg = xcat.float().reshape(outer, rows, C).permute(0, 2, 1).requires_grad_(True)
    r2 = F.group_norm(xg, 32, gamma, beta, 1e-5)
    if silu:
        r2 = F.silu(r2)
    r2.backward(dy.float().view(outer, rows, C).permute(0, 2, 1))
    dxr = xg.grad.permute(0, 2, 1).reshape(outer * rows, C)
    _close(dx1, dxr[:, :C1], what="groupnorm dx (fused stats)")
    if C2:
        _close(dx2, dxr[:, C1:], what="groupnorm dx2 (fused stats)")


@pytest.mark.parametrize("world,rank", [(1, 0), (2, 1), (3, 1), (8, 5)])
def test_adamw_p2p_kernel_matches_reduce_scatter_adamw_all_gather(raw, world, rank):
    """svdx_adamw_step_p2p on one device (the 'peer' arenas are local tensors): slice [lo, hi) of the summed gradients goes through
    AdamW and lands as bf16 in EVERY shadow arena; everything outside the slice stays untouched. Reference: svdx_adamw_step on
    the summed gradient slice (what reduce-scatter -> AdamW -> all-gather computes)."""
    n_total = 4096 * world
    n = n_total // world
    lo = rank * n
    grads = [_rand(n_total, seed=30 + r) for r in range(world)]
    shadows = [torch.full((n_total,), 7.0, device=DEV, dtype=bf16) for _ in range(world)]
    data = _rand(n_total, seed=50)
    p = data[lo:lo + n].clone()
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    state = torch.tensor([1e-2, 0.9, 0.999, 1e-8, 1e-2, 0.0, 1.0, 1.0], device=DEV)
    p_ref, m_ref, v_ref, state_ref = p.clone(), m.clone(), v.clone(), state.clone()
    sh_ref = torch.empty(n, device=DEV, dtype=bf16)
    for _ in range(3):
        raw.adamw_p2p(p, m, v, grads, shadows, lo, state, 1.0 / world)
        gsum = grads[0][lo:lo + n].clone()
        for r in range(1, world):
            gsum += grads[r][lo:lo + n]
        raw.adamw_graph(p_ref, gsum, m_ref, v_ref, state_ref, 1.0 / world, shadow=sh_ref)
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref) and torch.equal(m, m_ref) and torch.equal(v, v_ref) and torch.equal(state, state_ref)
    for r in range(world):
        assert torch.equal(shadows[r][lo:lo + n], sh_ref)
        rest = torch.cat([shadows[r][:lo], shadows[r][lo + n:]])
        assert bool((rest == 7.0).all())
    # launch accounting: tick + update, or the update alone
    counts = []
    for tick in (True, False):
        l0 = raw.LAUNCHES[0]
        raw.adamw_p2p(p, m, v, grads, shadows, lo, state, 1.0 / world, tick=tick)
        counts.append(raw.LAUNCHES[0] - l0)
    assert counts == [2, 1]
