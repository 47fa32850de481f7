"""GPU parity at the BASELINE shapes (round 2; VERDICT r1 "next" #1): the code paths the benchmark runs — 128 x 256 / 256 x 128 GEMM
tiles, hyper-connection kernels at D = 512 / 1024, wgmma attention at N' = 1056 with 8 heads, the whole d512 / depth-8 model and
a d1024 / 16-head model — against the fp32 oracle (oracle/e2tts_oracle.py) computed on the box's CPU inside the test, never against
a sibling kernel. All calls go through the C ABI. Tolerances as in test_gpu_parity.py (bf16 tensor-core path vs fp32 oracle).
"""
import pytest
import torch
import torch.nn.functional as F

from attn_ref import dropout_keep
from conftest import rel_l2
from kernel_checks import dev, pkg
from model_checks import check, cos, sample_vs_oracle, small_model, whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


def bf(t):
    return t.to(torch.bfloat16).contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# (c) every GEMM tile configuration, at sizes where the auto-selection of the benchmark picks it, incl. all epilogues
@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
def test_gemm_tiles_and_epilogues(pkg, force_tile):
    torch.manual_seed(10 + force_tile)
    ops = pkg.ops
    M, N, K = 1096, 520, 320        # ragged in M and N: partial tiles in both directions for every tile shape
    A, B = bf(torch.randn(M, K, device=dev())), bf(torch.randn(N, K, device=dev()) * 0.1)
    ref = A.float() @ B.float().t()
    kw = dict(force_tile=force_tile)
    check('plain', ops.gemm(A, B, M, N, K, **kw)[:, :N], ref, 1e-2)
    At, Bt = A.t().contiguous(), B.t().contiguous()
    check('b mn-major', ops.gemm(A, Bt, M, N, K, b_mn=True, **kw)[:, :N], ref, 1e-2)
    check('a mn-major', ops.gemm(At, B, M, N, K, lda=M, a_mn=True, **kw)[:, :N], ref, 1e-2)
    got = ops.gemm(At, Bt, M, N, K, lda=M, ldb=N, a_mn=True, b_mn=True, out_fp32=True, split_k=3, **kw)
    check('dW split-k', got, ref, 1e-3)
    got = ops.gemm(At, Bt, M, N, K, lda=M, ldb=N, a_mn=True, b_mn=True, out_fp32=True, **kw)
    check('fp32 out', got, ref, 1e-3)
    A1, A2 = A[:, :192].contiguous(), A[:, 192:].contiguous()
    check('two-source', ops.gemm(A1, B, M, N, K, lda=192, A2=A2, lda2=128, K1=192, **kw)[:, :N], ref, 1e-2)
    # fused epilogue: bias, per-batch column gate (rows_per_batch not a multiple of 32: warps straddle batch elements), row mask, residual
    rpb = 274
    bias = torch.randn(N, device=dev())
    cs = torch.rand(M // rpb, N, device=dev()) + 0.5
    mask = (torch.rand(M, device=dev()) > 0.2).to(torch.uint8)
    resid = bf(torch.randn(M, N + 0, device=dev()))
    ldr = (N + 7) // 8 * 8
    resid_p = torch.zeros(M, ldr, device=dev(), dtype=torch.bfloat16)
    resid_p[:, :N] = resid
    want = (ref + bias) * cs.repeat_interleave(rpb, 0) * mask[:, None].float() + resid.float()
    got = ops.gemm(A, B, M, N, K, bias=bias, colscale=cs, rows_per_batch=rpb, rowmask=mask, resid=resid_p, ldr=ldr, **kw)[:, :N]
    check('epilogue', got, want, 1e-2)
    # GEGLU (N multiple of 128, packed [u(64) | gate(64)] rows) with the saved pre-activations
    N2 = 512
    W = bf(torch.randn(N2, K, device=dev()) * 0.1)
    b2 = torch.randn(N2, device=dev()) * 0.1
    ug = torch.empty(M, N2, device=dev(), dtype=torch.bfloat16)
    h = ops.gemm(A, W, M, N2, K, D2=ug, ldd2=N2, bias=b2, geglu=True, **kw)
    z = A.float() @ W.float().t() + b2
    zz = z.view(M, N2 // 128, 2, 64)
    want_h = (zz[:, :, 0] * F.gelu(zz[:, :, 1])).reshape(M, N2 // 2)
    check('geglu pre-activations', ug, z, 1e-2)
    check('geglu', h[:, :N2 // 2], want_h, 1.5e-2)


# ----------------------------------------------------------------------------------------------------------------------
# (b) hyper-connection width/depth at every template instantiation: D = 128/256 (<1,*>), 512 (<2,*>, the benchmark), 1024 (<4,false>),
#     with enough tokens that every warp of the persistent forward grid walks several tokens (prefetch double buffer wraps)
@pytest.mark.parametrize('D', [128, 256, 512, 1024])
def test_hyper_width_depth_all_widths(pkg, D):
    torch.manual_seed(20 + D)
    ops = pkg.ops
    B, n, S = 2, 1300, 4
    T = B * n
    x = (torch.randn(T, S, D, device=dev()) * 1.5).to(torch.bfloat16).requires_grad_()
    P = dict(gamma=torch.randn(D) * 0.1, afn=torch.randn(D, S + 1) * 0.05, ascale=torch.tensor(0.5), salpha=torch.randn(S, S + 1) * 0.5 + 0.3,
             bfn=torch.randn(D) * 0.05, bscale=torch.tensor(0.7), sbeta=torch.randn(S) * 0.3 + 1)
    P = {k: v.to(dev()).requires_grad_() for k, v in P.items()}
    gain = (1 + 0.2 * torch.randn(B, D, device=dev())).requires_grad_()
    y = bf(torch.randn(T, D, device=dev())).requires_grad_()
    for mode, ng in ((2, gain), (1, gain[0].detach().clone().requires_grad_()), (0, None)):
        br, res, beta = ops.HcWidth.apply(x, P['gamma'], P['afn'], P['ascale'], P['salpha'], P['bfn'], P['bscale'], P['sbeta'], ng, mode, n)
        out = ops.HcDepth.apply(res, y, beta)
        wb, wo = torch.randn_like(br, dtype=torch.float32), torch.randn_like(out, dtype=torch.float32)
        loss = (br.float() * wb).sum() + (out.float() * wo).sum()
        leaves = [x, y] + list(P.values()) + ([ng] if ng is not None else [])
        grads = torch.autograd.grad(loss, leaves)
        xr = x.detach().float().cpu().view(B, n, S, D).requires_grad_()
        yr = y.detach().float().cpu().view(B, n, D).requires_grad_()
        sd = {'p.norm.gamma': P['gamma'], 'p.dynamic_alpha_fn': P['afn'], 'p.dynamic_alpha_scale': P['ascale'], 'p.static_alpha': P['salpha'],
              'p.dynamic_beta_fn': P['bfn'], 'p.dynamic_beta_scale': P['bscale'], 'p.static_beta': P['sbeta']}
        sd = {k: v.detach().cpu().clone().requires_grad_() for k, v in sd.items()}
        ngr = ng.detach().cpu().clone().requires_grad_() if ng is not None else None
        b0, rest, be = O.hyper_width(sd, 'p', xr, S)
        if mode == 2:
            b0 = F.normalize(b0, dim=-1) * D ** 0.5 * ngr[:, None, :]
        elif mode == 1:
            b0 = F.normalize(b0, dim=-1) * D ** 0.5 * ngr
        o = O.hyper_depth(rest, be, yr)
        lr = (b0 * wb.cpu().view(B, n, D)).sum() + (o * wo.cpu().view(B, n, S, D)).sum()
        rleaves = [xr, yr] + list(sd.values()) + ([ngr] if ng is not None else [])
        rgrads = torch.autograd.grad(lr, rleaves)
        check(f'branch m{mode}', br, b0.reshape(T, D), 2e-2)
        check(f'out m{mode}', out, o.reshape(T, S, D), 2e-2)
        check(f'beta m{mode}', beta, be.reshape(T, S), 1e-3)
        names = ['d_xres', 'd_y', 'gamma', 'afn', 'ascale', 'salpha', 'bfn', 'bscale', 'sbeta', 'gain']
        for nm, a, b in zip(names, grads, rgrads):
            check(f'{nm} m{mode} D{D}', a.reshape(-1), b.reshape(-1), 3e-2)


# (b') the depth connection of sub-block k fused into the width connection of sub-block k+1 (ops.HcDepthWidth): forward outputs and every
#      gradient — d residual', d branch_out, d beta of the folded depth connection and all parameter gradients (the parameter GEMM runs on
#      two K sources, residual' rows then branch rows) — against the oracle's hyper_depth followed by hyper_width
@pytest.mark.parametrize('D', [128, 256, 512, 1024])
def test_hyper_depth_width_fused(pkg, D):
    torch.manual_seed(40 + D)
    ops = pkg.ops
    B, n, S = 2, 1312, 4          # T * S = 10496 = 64 * 164
    T = B * n
    assert ops.hc_can_fuse(T, S)
    rest = (torch.randn(T, S, D, device=dev()) * 1.5).to(torch.bfloat16).requires_grad_()
    yp = bf(torch.randn(T, D, device=dev())).requires_grad_()
    bp = (1 + 0.3 * torch.randn(T, S, device=dev())).requires_grad_()
    P = dict(gamma=torch.randn(D) * 0.1, afn=torch.randn(D, S + 1) * 0.05, ascale=torch.tensor(0.5), salpha=torch.randn(S, S + 1) * 0.5 + 0.3,
             bfn=torch.randn(D) * 0.05, bscale=torch.tensor(0.7), sbeta=torch.randn(S) * 0.3 + 1)
    P = {k: v.to(dev()).requires_grad_() for k, v in P.items()}
    gain = (1 + 0.2 * torch.randn(B, D, device=dev())).requires_grad_()
    for mode, ng in ((2, gain), (0, None)):
        br, res, beta = ops.HcDepthWidth.apply(rest, yp, bp, P['gamma'], P['afn'], P['ascale'], P['salpha'], P['bfn'], P['bscale'], P['sbeta'], ng, mode, n)
        wb, wr, wbe = torch.randn_like(br, dtype=torch.float32), torch.randn_like(res, dtype=torch.float32), torch.randn_like(beta)
        loss = (br.float() * wb).sum() + (res.float() * wr).sum() + (beta * wbe).sum()
        leaves = [rest, yp, bp] + list(P.values()) + ([ng] if ng is not None else [])
        grads = torch.autograd.grad(loss, leaves)
        rr = rest.detach().float().cpu().view(B, n, S, D).requires_grad_()
        yr = yp.detach().float().cpu().view(B, n, D).requires_grad_()
        br_ = bp.detach().cpu().view(B, n, S).requires_grad_()
        sd = {'p.norm.gamma': P['gamma'], 'p.dynamic_alpha_fn': P['afn'], 'p.dynamic_alpha_scale': P['ascale'], 'p.static_alpha': P['salpha'],
              'p.dynamic_beta_fn': P['bfn'], 'p.dynamic_beta_scale': P['bscale'], 'p.static_beta': P['sbeta']}
        sd = {k: v.detach().cpu().clone().requires_grad_() for k, v in sd.items()}
        ngr = ng.detach().cpu().clone().requires_grad_() if ng is not None else None
        x_in = O.hyper_depth(rr, br_, yr)                     # the streams the fused kernel never writes out
        b0, rst, be = O.hyper_width(sd, 'p', x_in, S)
        if mode == 2:
            b0 = F.normalize(b0, dim=-1) * D ** 0.5 * ngr[:, None, :]
        lr = (b0 * wb.cpu().view(B, n, D)).sum() + (rst * wr.cpu().view(B, n, S, D)).sum() + (be * wbe.cpu().view(B, n, S)).sum()
        rleaves = [rr, yr, br_] + list(sd.values()) + ([ngr] if ng is not None else [])
        rgrads = torch.autograd.grad(lr, rleaves)
        check(f'branch m{mode}', br, b0.reshape(T, D), 2e-2)
        check(f'res m{mode}', res, rst.reshape(T, S, D), 2e-2)
        check(f'beta m{mode}', beta, be.reshape(T, S), 1e-3)
        names = ['d_rest', 'd_y_prev', 'd_beta_prev', 'gamma', 'afn', 'ascale', 'salpha', 'bfn', 'bscale', 'sbeta', 'gain']
        for nm, a, b in zip(names, grads, rgrads):
            check(f'{nm} m{mode} D{D}', a.reshape(-1), b.reshape(-1), 3e-2)


# ----------------------------------------------------------------------------------------------------------------------
# (d) wgmma attention core against an fp32 softmax written here (x-transformers Attend as the reference configures it, SURVEY A.4
#     steps 4-5: scale, tanh soft clamp 50, key-padding mask, fp32 softmax, dropout, per-head gate), at the benchmark's sequence length
#     and at short, unmasked and dropout cases
def _attn_core_ref(q, k, v, gate, mask, clamp=50.0, dropout=0.0, seed=0):
    """-> og [B*Np, H*dh] (gated, head-merged), o [B, H, Np, dh], lse [B, H, Np] (log-sum-exp of the clamped, masked logits). With
    dropout the kept probabilities are scaled by 65536 / (65536 - thresh16), the kernels' exact 1 / (1 - p)."""
    B, H, Np, dh = q.shape
    sim = torch.einsum('bhid,bhjd->bhij', q, k) * dh ** -0.5
    sim = torch.tanh(sim / clamp) * clamp
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], -torch.finfo(sim.dtype).max)
    attn = torch.softmax(sim, dim=-1)
    if dropout > 0:
        thresh16 = int(dropout * 65536)
        attn = attn * dropout_keep(seed, B, H, Np, dropout) * (65536 / (65536 - thresh16))
    o = torch.einsum('bhij,bhjd->bhid', attn, v)
    og = o * gate.view(B, Np, H).permute(0, 2, 1)[..., None]
    return og.permute(0, 2, 1, 3).reshape(B * Np, H * dh), o, torch.logsumexp(sim, dim=-1)


@pytest.mark.parametrize('Np,H,big_logits,masked,dropout', [
    (1056, 8, False, True, 0.0), (1056, 8, True, True, 0.0), (2080, 16, False, True, 0.0), (331, 3, True, True, 0.0),
    (128, 3, False, False, 0.0), (300, 3, False, True, 0.0), (1056, 3, False, True, 0.1), (40, 3, False, True, 0.0), (65, 2, False, False, 0.0)],
    ids=['1056-8-False', '1056-8-True', '2080-16-False', '331-3-True', '128-3-unmasked', '300-3-masked', '1056-3-masked-dropout', '40-3-masked',
         '65-2-unmasked'])
def test_attention_core_vs_fp32_softmax(pkg, Np, H, big_logits, masked, dropout):
    torch.manual_seed(30 + Np + H)
    ops = pkg.ops
    B = 2 if Np < 2000 else 1
    s = 3.0 if big_logits else 1.0      # big_logits: |q.k|/8/50 beyond the polynomial-tanh range -> the MUFU.TANH path
    q, k, v = (bf(torch.randn(B, H, Np, 64, device=dev()) * (s if i < 2 else 1.0)) for i in range(3))
    gate = torch.rand(B * Np, H, device=dev())
    m = torch.ones(B, Np, dtype=torch.bool, device=dev())
    if masked:
        m[0, Np // 3: Np // 3 + 40] = False
        m[B - 1, Np - 29:] = False
    mask = m.to(torch.uint8).contiguous() if masked else None
    seed = 4242
    og, o, lse = ops._attn_core_fwd(q, k, v, gate, mask, dropout, seed, 50.0, None)
    leaves = [t.clone().requires_grad_() for t in (q, k, v)] + [gate.clone().requires_grad_()]
    og_g = ops.AttnCore.apply(*leaves, mask, dropout, seed, 50.0, None)
    w = bf(torch.randn(B * Np, H * 64, device=dev()))
    grads = torch.autograd.grad(og_g, leaves, w)
    rl = [t.detach().float().cpu().requires_grad_() for t in leaves]
    ref_og, ref_o, ref_lse = _attn_core_ref(*rl, m.cpu(), dropout=dropout, seed=seed)
    rgrads = torch.autograd.grad(ref_og, rl, w.float().cpu())
    check('attention out', og, ref_og, 1e-2)
    assert torch.equal(og_g, og)
    check('attention o', o, ref_o, 1e-2)
    lse_err = float((lse.cpu() - ref_lse.detach()).abs().max())
    assert lse_err < 2e-2, f'attention lse: max abs error {lse_err:.4g}'
    for nm, a, b in zip(['dq', 'dk', 'dv', 'dgate'], grads, rgrads):
        check(f'attention {nm}', a, b, 2e-2)


# ----------------------------------------------------------------------------------------------------------------------
# (a), (e) whole model at the BASELINE widths against the oracle run on the host CPU
def test_e2tts_cfg2_shape_vs_oracle(pkg):
    """BASELINE cfg2's model (d512, depth 8, 8 heads) at its sequence length (N = 1024, N' = 1056), B = 2 with a ragged batch:
    T = 2112 rows -> the 128 x 256 GEMM tile, hc_width_*<2,true>, 9-tile wgmma attention — what bench.py times."""
    whole_model(pkg, dict(dim=512, depth=8, heads=8), B=2, N=1024, lens=[1024, 800], seed=40)


def test_e2tts_cfg3_kernels_vs_oracle(pkg):
    """cfg3 / cfg5's width (d1024, 16 heads, dim_text 512) at N = 2048 (N' = 2080): hc_width_*<4,false>, 16-head qkv packing,
    17-tile attention; depth 2 keeps the host oracle within seconds."""
    whole_model(pkg, dict(dim=1024, depth=2, heads=16), B=1, N=2048, lens=[1900], seed=50)


def test_e2tts_attn_fourier_embed_input_vs_oracle(pkg):
    """SURVEY §8f row 4, first variant: Transformer(attn_fourier_embed_input=True) (e2_tts.py:545-546; LinearFourierEmbed :368-386 on the
    attention input, :909) — wgmma GEMM + b200_fourier_feat_* against the oracle, which tests/test_oracle_vs_reference.py pins to the
    reference's own code with the switch on. Loss, prediction and every parameter gradient incl. `layers.{i}.0.4.linear.weight`."""
    whole_model(pkg, dict(dim=256, depth=2, heads=4, attn_fourier_embed_input=True), B=2, N=224, lens=[224, 170], seed=60)


def test_e2tts_concat_cond_vs_oracle(pkg):
    """SURVEY §8f row 4, third variant: E2TTS(concat_cond=True) (e2_tts.py:1134, :1200-1201, :1263-1267): the stem GEMM reads
    cat(cond, x) (b200_stem_prepare concat layout) against ONE packed Linear(2C -> dim); oracle pinned to the reference's own code."""
    whole_model(pkg, dict(dim=256, depth=2, heads=4), B=2, N=224, lens=[224, 190], seed=80, e2tts_kw=dict(concat_cond=True))


def test_e2tts_interpolated_text_vs_oracle(pkg):
    """SURVEY §8f row 4, second variant: E2TTS(interpolated_text=True) (e2_tts.py:1135, :1233; InterpolatedCharacterEmbed :414-482) —
    b200_interp_text_* + the abs-pos Linear as a wgmma GEMM with bias / residual / row-mask epilogue, against the oracle (pinned to
    the reference's own code in tests/test_oracle_vs_reference.py): ragged text and audio lengths, gradients of the embedding table
    and both abs_pos_mlp linears included."""
    whole_model(pkg, dict(dim=256, depth=2, heads=4), B=2, N=224, lens=[224, 150], seed=70, e2tts_kw=dict(interpolated_text=True))


# ----------------------------------------------------------------------------------------------------------------------
# (f) sampling: euler, 32 steps, autoguidance null model — against the oracle's fixed-grid ODE on the host
SMALL = dict(dim=128, depth=2, heads=2)


def test_sample_32_steps_vs_oracle(pkg):
    sample_vs_oracle(pkg, 60, SMALL)


def test_sample_euler_and_null_model(pkg):
    """odeint method 'euler' (e2_tts.py:1122-1126 odeint_kwargs) and `cfg_null_model` autoguidance (:1318-1321: the null prediction
    comes from a second, weaker model WITH text instead of this model without text)."""
    model, sd = small_model(pkg, 70, **SMALL)
    cfg = O.TransformerCfg(**SMALL)
    weak, wsd = small_model(pkg, 80, **SMALL)
    model.odeint_kwargs = dict(method='euler')
    torch.manual_seed(71)
    cond = torch.randn(2, 20, 100)
    text = ['Hello', 'Goodbye']
    tid = O.list_str_to_tensor(text)
    y0 = torch.randn(2, 48, 100)
    steps, strength = 6, 1.5
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(cond.to(dev()), text=text, duration=48, steps=steps, cfg_strength=strength, cfg_null_model=weak, return_raw_output=True)
    # host restatement of the same loop with the oracle's pieces (euler on linspace(0, 1, steps), SURVEY A.7)
    with torch.no_grad():
        lens = torch.maximum((tid != -1).sum(-1), torch.full((2,), 20))
        cond_mask = F.pad(O.lens_to_mask(lens, int(lens.amax())), (0, 48 - int(lens.amax())), value=False)[..., None]
        condp = F.pad(cond, (0, 0, 0, 48 - 20))
        step_cond = torch.where(cond_mask, condp, torch.zeros_like(condp))
        mask = O.lens_to_mask(torch.full((2,), 48), 48)
        ts = torch.linspace(0, 1, steps)
        y = y0
        for i in range(steps - 1):
            pred = O.transformer_with_pred_head(sd, cfg, y, step_cond, ts[i], mask, tid, False)
            null = O.transformer_with_pred_head(wsd, cfg, y, step_cond, ts[i], mask, tid, False)
            _, orth = O.project(pred - null, pred)
            y = y + (ts[i + 1] - ts[i]) * (pred + orth * strength)
        want = torch.where(cond_mask, condp, y)
    assert rel_l2(out.cpu(), want) < 5e-2


# ----------------------------------------------------------------------------------------------------------------------
# SURVEY §8f row 2: velocity-consistency loss (e2_tts.py:1556-1576; trainer hook trainer.py:259-268) — a second, no-grad forward of the
# EMA model at t + delta through the same kernels, fused into the loss head
def test_velocity_consistency_loss_vs_oracle(pkg):
    model, sd = small_model(pkg, 90, **SMALL)
    cfg = O.TransformerCfg(**SMALL)
    ema, esd = small_model(pkg, 91, **SMALL)
    ema.eval()
    model.train()
    model.velocity_consistency_weight = 0.7
    torch.manual_seed(92)
    B, N = 2, 96
    mel = torch.randn(B, N, 100)
    text = ['Hello', 'Goodbye']
    lens = torch.tensor([96, 70])
    x0, times = torch.randn(B, N, 100), torch.rand(B) * 0.9
    span = torch.zeros(B, N, dtype=torch.bool)
    span[:, 10:60] = True
    with pkg.inject_randomness(x0=x0.to(dev()), times=times.to(dev()), span_mask=span.to(dev()), drop_text_cond=False):
        out = model(mel.to(dev()), text=text, lens=lens.to(dev()), velocity_consistency_model=ema, velocity_consistency_delta=1e-3)
    out.loss.backward()
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = O.e2tts_forward(osd, cfg, mel, O.list_str_to_tensor(text), x0=x0, times=times, span_mask=span, lens=lens, velocity_sd=esd,
                          velocity_consistency_weight=0.7, velocity_consistency_delta=1e-3)
    ref['loss'].backward()
    assert abs(float(out.loss) - float(ref['loss'])) <= 1e-2 * abs(float(ref['loss']))
    assert abs(float(out.loss_breakdown.flow) - float(ref['flow_loss'])) <= 1e-2 * abs(float(ref['flow_loss']))
    assert abs(float(out.loss_breakdown.velocity_consistency) - float(ref['velocity_loss'])) <= 2e-2 * abs(float(ref['velocity_loss']))
    assert float(ref['velocity_loss']) > 0.1 * float(ref['flow_loss'])      # the term matters in this case
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None or float(gr.norm()) < 1e-4 * total:
            continue
        assert cos(p.grad.cpu(), gr) >= 0.99, k
    assert all(p.grad is None for p in ema.parameters())
    # without a velocity model the breakdown's second entry is the zero buffer, as in the reference (:1554)
    with pkg.inject_randomness(x0=x0.to(dev()), times=times.to(dev()), span_mask=span.to(dev()), drop_text_cond=False):
        out2 = model(mel.to(dev()), text=text, lens=lens.to(dev()))
    assert float(out2.loss_breakdown.velocity_consistency) == 0.0
    assert abs(float(out2.loss) - float(ref['flow_loss'])) <= 1e-2 * abs(float(ref['flow_loss']))


# ----------------------------------------------------------------------------------------------------------------------
# SURVEY §8f row 3: on-device data path — MelSpec per item (trainer.py:101-131) + collate_fn (:61-82) + 'b d n -> b n d' (:253) as one launch
def test_melspec_collate_ragged_batch_vs_per_item_reference(pkg):
    torch.manual_seed(100)
    ms = pkg.MelSpec().to(dev())
    lens = [256 * 24, 256 * 17 + 100, 5000, 256 * 24 - 1]
    waves = [torch.randn(n) * 0.3 for n in lens]
    batch = ms.collate(waves)
    per_item = [O.melspec(w[None])[0] for w in waves]                 # [n_mels, frames_i] each (torchaudio semantics, pinned by test_oracle_*)
    n_max = max(m.shape[-1] for m in per_item)
    want = torch.stack([F.pad(m, (0, n_max - m.shape[-1])) for m in per_item]).transpose(1, 2)   # collate_fn zero-pads, trainer transposes
    assert batch['mel'].shape == want.shape, (batch['mel'].shape, want.shape)
    assert batch['mel_lengths'].tolist() == [m.shape[-1] for m in per_item]
    assert float((batch['mel'].cpu() - want).abs().max()) < 1e-3
    # the batched output feeds the model directly
    model = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), use_vocos=False).to(dev())
    out = model(batch['mel'], text=['a', 'b', 'c', 'd'], lens=batch['mel_lengths'])
    assert torch.isfinite(out.loss)
    # a long wave at the benchmark's frame count (1024 frames) against the oracle
    wave = torch.randn(2, 256 * 1023) * 0.2
    got = ms(wave.to(dev()))
    assert got.shape == (2, 100, 1024)
    assert float((got.cpu() - O.melspec(wave)).abs().max()) < 1e-3
