"""Decoder-head, contrastive, pixel-target and AdamW kernels against the golden fixtures and the oracle (gpu).  The token
front end is tested in test_embed_gpu.py."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import restate

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.mark.parametrize("M,C", [(50, 3200), (417, 1408), (9, 768), (130, 160)])
@pytest.mark.parametrize("tf32", [True, False])
def test_ln_l2_and_align_loss(cuda_lib, M, C, tf32):
    ll = cuda_lib
    torch.manual_seed(M)
    z = (torch.randn(M, C, device="cuda") * 1.5 + 0.2).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(C, device="cuda")).to(torch.bfloat16)
    b = (0.1 * torch.randn(C, device="cuda")).to(torch.bfloat16)
    tgt = torch.nn.functional.normalize(torch.randn(M, C, device="cuda"), dim=-1)
    if not tf32:
        tgt = tgt.to(torch.bfloat16)
    zr = z.float().requires_grad_(True); wr = w.float().requires_grad_(True); br = b.float().requires_grad_(True)
    out_ref = restate.l2n(restate.layernorm(zr, wr, br))
    loss_ref = restate.align_loss(out_ref, tgt.float())
    ls = torch.zeros(1, device="cuda")
    out, stats = ll.ln_l2_fwd(z, w, b, 1e-5, want_out=True, target=tgt, loss_sum=ls)
    assert _rel(out, out_ref) < 5e-3
    assert abs(ls.item() / M - loss_ref.item()) < 2e-4 * max(1.0, abs(loss_ref.item()))
    loss_ref.backward()
    dw = torch.zeros(C, device="cuda"); db = torch.zeros(C, device="cuda")
    g = torch.full((1,), 1.0, device="cuda")
    dz = ll.ln_l2_bwd(z, w, b, stats, tgt, gscale_host=-2.0 / M, gscale_dev=g, dweight=dw, dbias=db)
    assert _rel(dz, zr.grad) < 8e-3
    assert _rel(dw, wr.grad) < 2e-3 and _rel(db, br.grad) < 2e-3


def test_vtc_against_golden_and_oracle(cuda_lib):
    ll = cuda_lib
    z = np.load(GOLD / "vtc.npz")
    v = torch.cat([torch.from_numpy(z["v0"]), torch.from_numpy(z["v1"])]).cuda()
    t = torch.cat([torch.from_numpy(z["t0"]), torch.from_numpy(z["t1"])]).cuda()
    idx = torch.cat([torch.from_numpy(z["idx0"]), torch.from_numpy(z["idx1"])]).cuda()
    temp = float(z["temp"])
    vn, vinv = ll.l2norm_rows_fwd(v); tn, tinv = ll.l2norm_rows_fwd(t)
    cosm = ll.gemm(vn, tn, epi=ll.EPI_F32)
    loss, lr_, lc_ = ll.vtc_loss_fwd(cosm, idx, temp)
    assert abs(loss.item() - float(z["loss0"])) < 3e-2          # bf16 embeddings at temp 0.07
    # fp32 check of the loss/grad kernels alone (cos from fp32 torch)
    vr = v.clone().requires_grad_(True); tr = t.clone().requires_grad_(True)
    cos32 = torch.nn.functional.normalize(vr, dim=-1) @ torch.nn.functional.normalize(tr, dim=-1).t()
    cos32.retain_grad()
    s = cos32 / temp
    tg = restate.get_mask(idx.cpu()).cuda()
    l_ref = (-(torch.log_softmax(s, 1) * tg).sum(1).mean() - (torch.log_softmax(s.t(), 1) * tg).sum(1).mean()) / 2
    l_ref.backward()
    loss2, lr2, lc2 = ll.vtc_loss_fwd(cos32.detach().contiguous(), idx, temp)
    assert abs(loss2.item() - l_ref.item()) < 1e-4
    assert abs(l_ref.item() - float(z["loss0"])) < 1e-4
    dcos, dtemp = ll.vtc_loss_bwd(cos32.detach().contiguous(), idx, temp, lr2, lc2)
    assert _rel(dcos, cos32.grad) < 6e-3
    # local-row input grads (AllGather.backward keeps the local slice): rank 0 rows
    dv_n = ll.gemm(dcos[:8].contiguous(), tn, b_t=True, epi=ll.EPI_F32)
    dv = ll.l2norm_rows_bwd(dv_n, vn[:8].contiguous(), vinv[:8].contiguous())
    assert _rel(dv.cpu(), torch.from_numpy(z["gv0"])) < 3e-2


def test_pixel_targets_and_mse(cuda_lib):
    ll = cuda_lib
    z = np.load(GOLD / "pixel_target.npz")
    im = torch.from_numpy(z["images"]).to(torch.bfloat16)
    mask = torch.from_numpy(z["mask"])
    B, N = mask.shape
    midx = torch.stack([torch.nonzero(mask[b]).flatten() for b in range(B)]).to(torch.int32).flatten().cuda()
    mean3 = torch.tensor(restate.IMAGENET_MEAN, device="cuda"); std3 = torch.tensor(restate.IMAGENET_STD, device="cuda")
    lab = ll.pixel_targets(im.cuda(), midx, 4, 2, 16, True, mean3, std3)
    ref = restate.pixel_targets(im.float(), mask, 16, 2, True).reshape(B * 4, -1)
    assert _rel(lab.cpu(), ref) < 1e-4
    lab_raw = ll.pixel_targets(im.cuda(), midx, 4, 2, 16, False, mean3, std3)
    assert _rel(lab_raw.cpu(), restate.pixel_targets(im.float(), mask, 16, 2, False).reshape(B * 4, -1)) < 1e-5
    pred = torch.randn_like(lab).to(torch.bfloat16)
    ls = torch.zeros(1, device="cuda"); dp = torch.empty_like(pred)
    ll.mse_loss(pred, lab, ls, gscale_host=1.0 / pred.numel(), dpred=dp)
    assert abs(ls.item() / pred.numel() - restate.mse_loss(pred.float(), lab).item()) < 1e-4
    assert _rel(dp, 2 * (pred.float() - lab) / pred.numel()) < 5e-3


def test_loss_sums_repeat_bit_for_bit(cuda_lib):
    """The alignment loss, the contrastive loss, dtemp and the MSE sum their CTAs' partials in a fixed order: two calls
    on the same inputs, each over hundreds of CTAs, give the same bits."""
    ll = cuda_lib
    torch.manual_seed(0)
    M, C, G, n = 13312, 1408, 1024, 1 << 24
    z = torch.randn(M, C, device="cuda").to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(C, device="cuda")).to(torch.bfloat16)
    b = (0.1 * torch.randn(C, device="cuda")).to(torch.bfloat16)
    tgt = torch.nn.functional.normalize(torch.randn(M, C, device="cuda"), dim=-1).to(torch.bfloat16)
    cosm = torch.nn.functional.normalize(torch.randn(G, 64, device="cuda"), dim=-1)
    cosm = (cosm @ cosm.t()).contiguous()
    idx = torch.randint(0, G // 2, (G,), device="cuda")
    pred = torch.randn(n, device="cuda").to(torch.bfloat16)
    label = torch.randn(n, device="cuda")

    def scalars():
        align = torch.zeros(1, device="cuda")
        ll.ln_l2_fwd(z, w, b, 1e-5, want_out=False, target=tgt, loss_sum=align)
        vtc, lse_r, lse_c = ll.vtc_loss_fwd(cosm, idx, 0.07)
        _, dtemp = ll.vtc_loss_bwd(cosm, idx, 0.07, lse_r, lse_c)
        mse = ll.mse_loss(pred, label, torch.zeros(1, device="cuda"))
        return torch.cat([align, vtc, dtemp, mse])

    first, second = scalars(), scalars()
    assert torch.equal(first.view(torch.int32), second.view(torch.int32)), (first.tolist(), second.tolist())


def test_adamw_matches_torch(cuda_lib):
    ll = cuda_lib
    torch.manual_seed(0)
    n = 10007
    p0 = torch.randn(n, device="cuda")
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
    master = p0.clone(); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    for step in range(1, 4):
        g = torch.randn(n, device="cuda").to(torch.bfloat16)
        ref.grad = g.float()
        opt.step()
        ll.adamw_step(master, m, v, g, pb, 1e-3, 0.9, 0.95, 1e-8, 0.05, step)
    assert torch.allclose(master, ref.data, atol=1e-6, rtol=1e-5)
    assert torch.equal(pb, master.to(torch.bfloat16))
