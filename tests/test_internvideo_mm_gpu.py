"""InternVideo-MM on the H100 (gpu):
  - ivb_dpe_ln_fwd element by element against an fp64 evaluation of the same inputs (oracle.internvideo_mm.dpe_ln):
    the L/14 taps at 8 and 16 frames and one frame, a narrow tap and an odd grid, fp32 and bf16 streams, padded pitches,
    the cls rows included; each output within one bf16 rounding (2^-8 relative) plus 2^-12; the same bits on a second
    call;
  - the model against tests/golden/internvideo_mm.npz (the unmodified reference's fp32 outputs): video features, the
    image-mode features of one-frame clips, return_all_feats, text features with EOTs at different positions and with
    masked_indices, each within 1e-2 relative (Frobenius), and the demo's zero-shot probabilities within 1e-2;
  - one L/14-size extractor tap (C = 1024, 16 heads, 8 frames of 16 x 16 patches) against the fp32 restatement;
  - a B/16 checkpoint of a randomly initialised reference VideoIntern, saved with the `clip.` prefix, through
    load_model: the demo's three-caption probabilities within 1e-2 of the reference's;
  - set_fp8_inference reaches the backbone and text blocks, and switching it off restores the bf16 output bit for bit.
"""
import pytest
import torch

from internvideo_b200 import internvideo_mm as mm
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M
from oracle import internvideo_mm as om

pytestmark = pytest.mark.gpu
bf = torch.bfloat16


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm())


def _tap_params(C, seed):
    g = torch.Generator().manual_seed(seed)
    w = (0.2 * torch.randn(C, 1, 3, 3, 3, generator=g)).to(bf)
    b, lb = ((0.05 * torch.randn(C, generator=g)).to(bf) for _ in range(2))
    lw = (1 + 0.1 * torch.randn(C, generator=g)).to(bf)
    return w, b, lw, lb


@pytest.mark.parametrize("T,H,W,C", [(8, 16, 16, 1024), (16, 16, 16, 1024), (1, 16, 16, 1024), (4, 4, 4, 128),
                                     (3, 5, 7, 64)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("padded", [False, True], ids=["dense", "padded"])
def test_dpe_ln_against_fp64(T, H, W, C, dtype, padded):
    N = 2
    M_ = N * T * (1 + H * W)
    g = torch.Generator().manual_seed(T * 1000 + H * 10 + W + C)
    x = (2 * torch.randn(M_, C, generator=g)).to(dtype)
    w, b, lw, lb = _tap_params(C, C + T)
    pad = 64 if padded else 0
    xd = torch.zeros(M_, C + pad, dtype=dtype, device="cuda")
    xd[:, :C] = x.cuda()
    xd = xd[:, :C]
    out = torch.full((M_, C + pad), float("nan"), dtype=bf, device="cuda")[:, :C] if padded else None
    dev = [t.cuda() for t in (w, b, lw, lb)]
    y = ll._dpe_ln_fwd(xd, *dev, 1e-5, N, T, H, W, out=out)
    ref = om.dpe_ln(x.double(), w.double(), b.double(), lw.double(), lb.double(), N, T, H, W)
    err = (y.double().cpu() - ref).abs()
    assert bool((err <= 2.0 ** -8 * ref.abs() + 2.0 ** -12).all()), float(err.max())
    y2 = ll._dpe_ln_fwd(xd, *dev, 1e-5, N, T, H, W, out=torch.empty_like(out) if padded else None)
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16))


@pytest.fixture(scope="module")
def model():
    om.register_narrow(mm.BACKBONES, mm.VisionTransformer)
    try:
        sd, z = om.load()
        m = mm.VideoIntern(**om.MODEL)
    finally:
        mm.BACKBONES.pop(om.NARROW, None)
    m.load_state_dict(sd, strict=True)
    return m.bfloat16().cuda().eval(), z


def _video(z):
    video, image = om.stored_inputs(z)
    return video.cuda().to(bf), image.cuda().to(bf)


def test_video_image_and_all_feats_match_reference(model):
    m, z = model
    video, image = _video(z)
    v = m.encode_video(video)
    assert v.shape == (om.B, om.MODEL["embed_dim"]) and _rel(v, torch.from_numpy(z["video"])) < 1e-2
    img = m.encode_video(image, mode="image")
    assert _rel(img, torch.from_numpy(z["image"])) < 1e-2
    v_all, stream = m.encode_video(video, return_all_feats=True)
    assert torch.equal(v_all, v)
    assert stream.shape == z["stream"].shape and _rel(stream, torch.from_numpy(z["stream"])) < 1e-2


def test_text_and_zero_shot_match_reference(model):
    m, z = model
    ids = torch.from_numpy(z["ids"]).cuda()
    t, t_all = m.encode_text(ids, return_all_feats=True)
    assert _rel(t, torch.from_numpy(z["text"])) < 1e-2 and _rel(t_all, torch.from_numpy(z["text_all"])) < 1e-2
    masked = m.encode_text(ids, masked_indices=torch.from_numpy(z["mask"]).cuda())
    assert _rel(masked, torch.from_numpy(z["text_masked"])) < 1e-2
    probs = om.zero_shot(m.encode_video(_video(z)[0]).float(), t[:om.N_CAND].float(), m.logit_scale.detach().float())
    assert float((probs.cpu() - torch.from_numpy(z["probs"])).abs().max()) < 1e-2


def test_l14_extractor_tap_against_restatement():
    N, T, Hg, C, H = 2, 8, 16, 1024, 16
    L = 1 + Hg * Hg
    torch.manual_seed(0)
    dec = mm.Extractor(C, H)
    dpe = torch.nn.Conv3d(C, C, 3, padding=1, groups=C)
    sd = {}
    with torch.no_grad():
        for name, p in list(dec.named_parameters()) + [("dpe." + k, p) for k, p in dpe.named_parameters()]:
            p.copy_(om.draw_param("visual.transformer.dec.0." + name, tuple(p.shape)))
            sd[name] = p.detach().clone()
    g = torch.Generator().manual_seed(1)
    h = torch.randn(N * T * L, C, generator=g)
    cls = 0.5 * torch.randn(N, C, generator=g)
    keys = om.dpe_ln(h, sd["dpe.weight"], sd["dpe.bias"], sd["ln_3.weight"], sd["ln_3.bias"], N, T, Hg, Hg)
    ref = om.extractor(cls, keys.reshape(N, T * L, C), sd, "", H)
    dec, dpe = dec.bfloat16().cuda().eval(), dpe.bfloat16().cuda()
    with torch.no_grad():
        k = ll._dpe_ln_fwd(h.cuda(), dpe.weight, dpe.bias, dec.ln_3.weight, dec.ln_3.bias, 1e-5, N, T, Hg, Hg)
        got = dec.forward_rows(cls.cuda(), k, T * L)
    assert _rel(k, keys) < 1e-2
    assert _rel(got - cls.cuda(), ref - cls) < 1e-2


def test_load_model_zero_shot_matches_reference(tmp_path):
    ref_mod, _ = om.import_mm()
    torch.manual_seed(0)
    ref = ref_mod.VideoIntern(embed_dim=512, vision_width=768, context_length=77, vocab_size=1000,
                              transformer_width=128, transformer_heads=2, transformer_layers=2, n_layers=4, n_dim=768,
                              n_head=12, t_size=8, backbone="vit_only_global_b16", return_list=[8, 9, 10, 11]).eval()
    path = tmp_path / "mm.ckpt"
    torch.save({"state_dict": {"clip." + k: v for k, v in ref.state_dict().items()}}, path)
    g = torch.Generator().manual_seed(2)
    video = torch.randn(1, 3, 8, 224, 224, generator=g).to(bf).float()
    ids = torch.zeros(3, 77, dtype=torch.long)
    for b, n in enumerate((5, 4, 6)):
        ids[b, 0], ids[b, 1:n + 1], ids[b, n + 1] = 998, torch.randint(1, 998, (n,), generator=g), 999
    with torch.no_grad():
        want = om.zero_shot(ref.encode_video(video), ref.encode_text(ids), ref.logit_scale)
    port = mm.load_model(str(path)).bfloat16().cuda()
    got = om.zero_shot(port.encode_video(video.cuda().to(bf)).float(), port.encode_text(ids.cuda()).float(),
                       port.logit_scale.detach().float())
    assert float((got.cpu() - want).abs().max()) < 1e-2


def test_fp8_inference_reaches_the_blocks(model):
    m, z = model
    video, _ = _video(z)
    ids = torch.from_numpy(z["ids"]).cuda()
    v0, t0 = m.encode_video(video), m.encode_text(ids)
    try:
        assert M.set_fp8_inference(m) == om.VISION["layers"] + om.MODEL["transformer_layers"]
        v8, t8 = m.encode_video(video), m.encode_text(ids)
        assert torch.isfinite(v8).all() and torch.isfinite(t8).all() and not torch.equal(v8, v0)
    finally:
        M.set_fp8_inference(m, enabled=False)
    assert torch.equal(m.encode_video(video), v0) and torch.equal(m.encode_text(ids), t0)


def test_masked_text_flags_an_out_of_range_id(model):
    m, z = model
    ids = torch.from_numpy(z["ids"]).cuda()
    ids[1, 3] = om.MODEL["vocab_size"]
    out = m.encode_text(ids, masked_indices=torch.from_numpy(z["mask"]).cuda())
    assert torch.isnan(out.float()).all()


def test_dpe_ln_wrapper_refuses_bad_operands():
    N, T, H, C = 1, 2, 2, 64
    x = torch.zeros(N * T * (1 + H * H), C, device="cuda")
    w, b, lw, lb = (t.cuda() for t in _tap_params(C, 0))
    with pytest.raises(ll._lib.IvbError, match="conv_b must be a contiguous"):
        ll._dpe_ln_fwd(x, w, b[:32], lw, lb, 1e-5, N, T, H, H)
    with pytest.raises(ll._lib.IvbError, match="ln_w must be a contiguous"):
        ll._dpe_ln_fwd(x, w, b, lw[::2], lb, 1e-5, N, T, H, H)
    with pytest.raises(ll._lib.IvbError, match="out must be"):
        ll._dpe_ln_fwd(x, w, b, lw, lb, 1e-5, N, T, H, H, out=torch.empty(4, C, device="cuda", dtype=bf))
    xb = torch.zeros(N * T * (1 + H * H), 2 * C, device="cuda", dtype=bf)
    with pytest.raises(ll._lib.IvbError, match="must not overlap"):
        ll._dpe_ln_fwd(xb[:, :C], w, b, lw, lb, 1e-5, N, T, H, H, out=xb[:, 32:32 + C])
