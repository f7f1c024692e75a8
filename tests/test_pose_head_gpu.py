"""GPU: the pose head (pose_head_kernel, kernels.cu: fp32 MLP 768 -> 512 -> 512 -> 512, fc_t / fc_rot / fc_conf, row
normalisation and the one-sided Jacobi SVD projection svd_orthogonalize_3x3) against a float64 restatement of
head_pose_s (oracle/sta_oracle.py:351-369), on random tokens, on planted 3x3 matrices, and on the pose tokens of the
bf16 and FP8 models for the 12-token golden.

Rotation bound.  R = V diag(1, 1, det(V U^T)) U^T is the special-orthogonal projection of A = normalize_rows(M)^T =
U S V^T.  To first order a perturbation dA moves it by ||dR||_F <= 2 ||dA||_F / g, where g = sigma2 + sigma3 when
det A > 0 and g = sigma2 - sigma3 when det A < 0: the derivative of the polar factor divides the skew part of
U^T dA V by sigma_i + sigma_j over the pairs (i, j), and the determinant flip turns sigma3 into -sigma3.  dA has two
sources:
  * the fp32 MLP: a dot product of K terms as the kernel sums them (K / 32 sequential terms per lane, five shuffle
    levels, the bias) costs at most (K / 32 + 8) 2^-24 of sum |w x| + |b|; the 2-norm of the error of each layer's input
    goes through the spectral norm of W (ReLU is 1-Lipschitz).  Normalising a row r divides its error by |r|.
  * the fp32 normalisation and Jacobi sweeps: 2^-18 in ||dA||_F (a few dozen ulps of ||A||_2 <= sqrt 3).
so |R - R64| <= 2 (||dA||_F + 2^-18) / g + 2^-21 per entry.  Tokens where this is vacuous (> 1) or where ||dA||_F is not
small against g (first order no longer holds) are skipped and counted."""
import math

import pytest
import torch
import torch.nn.functional as F

from test_model_gpu import golden_case

pytestmark = pytest.mark.gpu

DEV = "cuda"
PFX = "head_pose_s."


def _gam(K):
    return (K / 32 + 8) * 2.0 ** -24


def head_pose64(sd, tok, tok_err=None):
    """float64 head_pose_s of dec_norm-ed tokens [B][768] from the fp32 weights, with first-order bounds on the fp32
    kernel's fc_t / fc_rot / fc_conf outputs; tok_err [B][768]: a bound on the error of the tokens the kernel starts
    from (its own fp32 dec_norm), zero if not given"""
    P = lambda k: sd[PFX + k].to(tok.device).double()  # noqa: E731
    x = tok.double()
    # 2-norm of the error of the layer input
    err = (torch.zeros(x.shape[0], device=x.device, dtype=torch.float64) if tok_err is None else
           tok_err.double().norm(dim=1))
    for i in (0, 2, 4):
        W, b = P("mlp.%d.weight" % i), P("mlp.%d.bias" % i)
        y = x @ W.t() + b
        rnd = _gam(W.shape[1]) * (x.abs() @ W.abs().t() + b.abs())
        err = torch.linalg.matrix_norm(W, ord=2) * err + rnd.norm(dim=1)
        x = y.clamp_min(0)

    def lin(name, rows):
        """outputs and, per group of `rows` outputs, the 2-norm of their error"""
        W, b = P(name + ".weight"), P(name + ".bias")
        rnd = _gam(512) * (x.abs() @ W.abs().t() + b.abs())
        Wg = W.view(-1, rows, 512)
        e = torch.linalg.matrix_norm(Wg, ord=2)[None, :] * err[:, None] + rnd.view(x.shape[0], -1, rows).norm(dim=2)
        return x @ W.t() + b, e

    t, et = lin("fc_t", 1)
    r9, er = lin("fc_rot", 3)
    c, ec = lin("fc_conf.0", 1)
    out = project64(r9.view(-1, 3, 3))
    rn = r9.view(-1, 3, 3).norm(dim=-1).clamp_min(1e-300)
    dA = ((er / rn + 2.0 ** -22) ** 2).sum(-1).sqrt()
    out.update(t=t, err_t=et + 2.0 ** -23 * t.abs(), conf=torch.sigmoid(c[:, 0]), err_conf=0.25 * ec[:, 0] + 2.0 ** -22,
               dA=dA)
    return out


def project64(M):
    """float64 svd_orthogonalize (pose_head.py:38-57) of M [B][3][3]: R, the singular values of A and det A"""
    A = F.normalize(M, p=2, dim=-1).transpose(-1, -2)
    u, s, vh = torch.linalg.svd(A)
    v = vh.transpose(-1, -2)
    d = torch.det(v @ u.transpose(-1, -2))
    R = torch.cat([v[:, :, :2], v[:, :, 2:] * d.view(-1, 1, 1)], dim=2) @ u.transpose(-1, -2)
    detA = torch.det(A)
    gap = torch.where(detA > 0, s[:, 1] + s[:, 2], s[:, 1] - s[:, 2])
    return {"R": R, "sig": s, "detA": detA, "gap": gap}


def rotation_bound(dA, gap):
    """per-token bound on |R - R64| (module docstring); inf where it is vacuous or not first order"""
    b = 2.0 * (dA + 2.0 ** -18) / gap.clamp_min(1e-300) + 2.0 ** -21
    return torch.where((b > 1.0) | (dA > 0.25 * gap), torch.full_like(b, math.inf), b)


def check_pose(name, pose, conf, ref):
    """kernel pose [B][4][4] / conf [B] against head_pose64's ref; returns (worst ratio, tokens skipped)"""
    P = pose.double()
    bound = rotation_bound(ref["dA"], ref["gap"])
    ok = torch.isfinite(bound)
    R = P[:, :3, :3]
    assert bool(torch.isfinite(P).all()), name + ": non-finite pose"
    so3 = (R @ R.transpose(1, 2) - torch.eye(3, dtype=R.dtype, device=R.device)).abs().amax((1, 2))
    assert float(so3.max()) < 1e-5 and float((torch.det(R) - 1).abs().max()) < 1e-5, name + ": R not in SO(3)"
    ratio_r = ((R - ref["R"]).abs().amax((1, 2)) / bound)[ok]
    ratio_t = ((P[:, :3, 3] - ref["t"]).abs() / ref["err_t"]).amax(1)
    ratio_c = (conf.double() - ref["conf"]).abs() / ref["err_conf"]
    worst = max(float(ratio_r.max()) if ratio_r.numel() else 0.0, float(ratio_t.max()), float(ratio_c.max()))
    skipped = int((~ok).sum())
    print("pose head %-36s worst err / bound = %.4f (rotation %.4f, t %.4f, conf %.4f); %d of %d tokens skipped "
          "(vacuous rotation bound)" % (name, worst, float(ratio_r.max()) if ratio_r.numel() else 0.0,
                                        float(ratio_t.max()), float(ratio_c.max()), skipped, P.shape[0]), flush=True)
    assert worst <= 1.0, name
    assert bool((P[:, 3] == torch.tensor([0, 0, 0, 1.0], dtype=P.dtype, device=P.device)).all())
    return worst, skipped


def test_pose_head_on_random_tokens_within_float64_bound(cuda_model, state_dict):
    g = torch.Generator(device=DEV).manual_seed(0)
    tok = torch.randn(4096, 768, generator=g, device=DEV)
    out = cuda_model.head_pose_s(tok)
    ref = head_pose64(state_dict, tok)
    _, skipped = check_pose("random tokens", out["pose"], out["conf"], ref)
    assert skipped < 4096 // 2, "most tokens skipped: the bound is not testing anything"


# ---------------------------------------------------------------------------------------------------------------------
# planted matrices: a pose-head-only model that routes token channels straight to fc_rot / fc_t / fc_conf
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def routed_model(state_dict):
    """mlp.0 row 2i = e_i, row 2i + 1 = -e_i (i < 13); mlp.2 and mlp.4 identities; fc_rot row j = e_2j - e_2j+1,
    fc_t row j = e_2(9+j) - e_2(9+j)+1, fc_conf = e_24 - e_25; zero biases.  Every dot product has one nonzero term, so
    token channels 0..8 reach fc_rot (row-major M), 9..11 fc_t and 12 fc_conf exactly."""
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    sd = dict(state_dict)
    w0 = torch.zeros(512, 768)
    for i in range(13):
        w0[2 * i, i], w0[2 * i + 1, i] = 1.0, -1.0
    sd[PFX + "mlp.0.weight"] = w0
    for i in (2, 4):
        sd[PFX + "mlp.%d.weight" % i] = torch.eye(512)
    for i in (0, 2, 4):
        sd[PFX + "mlp.%d.bias" % i] = torch.zeros(512)

    def rows(first, n):
        w = torch.zeros(n, 512)
        for j in range(n):
            w[j, 2 * (first + j)], w[j, 2 * (first + j) + 1] = 1.0, -1.0
        return w

    sd[PFX + "fc_rot.weight"], sd[PFX + "fc_rot.bias"] = rows(0, 9), torch.zeros(9)
    sd[PFX + "fc_t.weight"], sd[PFX + "fc_t.bias"] = rows(9, 3), torch.zeros(3)
    sd[PFX + "fc_conf.0.weight"], sd[PFX + "fc_conf.0.bias"] = rows(12, 1), torch.zeros(1)
    m = STA()
    m.load_state_dict(sd, strict=True)
    m.eval()
    return m


def _rot(axis, deg):
    a = torch.tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    K = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], dtype=torch.float64)
    th = math.radians(deg)
    return torch.eye(3, dtype=torch.float64) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


def _signed_permutations():
    import itertools
    out = []
    for p in itertools.permutations(range(3)):
        for s in itertools.product((1.0, -1.0), repeat=3):
            M = torch.zeros(3, 3, dtype=torch.float64)
            for i in range(3):
                M[i, p[i]] = s[i]
            if torch.det(M) > 0:
                out.append(M)
    return out


def _random_rotation(g):
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    return q if torch.det(q) > 0 else -q


def _planted_cases():
    g = torch.Generator().manual_seed(3)
    rot = [("identity", torch.eye(3, dtype=torch.float64)), ("rz90", _rot((0, 0, 1), 90)),
           ("180_about_x", _rot((1, 0, 0), 180)), ("180_about_110", _rot((1, 1, 0), 180)),
           ("180_about_111", _rot((1, 1, 1), 180)), ("120_about_111", _rot((1, 1, 1), 120))]
    rot += [("signed_perm%d" % i, M) for i, M in enumerate(_signed_permutations())]
    rot += [("random_rot%d" % i, _random_rotation(g)) for i in range(8)]
    # (name, M, kind): exact = R must equal the rotation, gap = first-order bound, so3 = only R in SO(3) and finite
    cases = [(n, M, "exact") for n, M in rot]
    cases += [("scaled_%s" % n, s * M, "exact") for n, M in rot[:6] for s in (3.7, 1e-3)]
    cases += [("row_scaled_%s" % n, torch.diag(torch.tensor([0.01, 5.0, 100.0], dtype=torch.float64)) @ M, "exact")
              for n, M in rot[6:12]]
    for i in range(6):
        M = _random_rotation(g) @ torch.diag(torch.tensor([1.0, 0.55, -0.2], dtype=torch.float64)) @ _random_rotation(g)
        cases.append(("reflection_gap%d" % i, M, "gap"))
        r = torch.randn(3, 3, generator=g, dtype=torch.float64)
        cases.append(("rank2_equal_rows%d" % i, torch.stack([r[0], r[0], r[2]]), "gap"))
        cases.append(("rank2_zero_row%d" % i, torch.stack([r[0], r[1], torch.zeros(3, dtype=torch.float64)]), "gap"))
        v = torch.randn(3, generator=g, dtype=torch.float64)
        cases.append(("rank1_%d" % i, torch.stack([v, 2 * v, -3 * v]), "so3"))
        cases.append(("reflection_equal_sigma%d" % i,
                      torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)) @ _random_rotation(g), "so3"))
    cases += [("rank1_axis", torch.tensor([[1.0, 0, 0]] * 3, dtype=torch.float64), "so3"),
              ("rank1_equal_rows", torch.tensor([[0.6, 0.0, 0.8]] * 3, dtype=torch.float64), "so3")]
    return cases


def test_planted_matrices_reach_the_svd_projection(routed_model):
    cases = _planted_cases()
    B = len(cases)
    M32 = torch.stack([M for _, M, _ in cases]).float()
    g = torch.Generator().manual_seed(4)
    t32 = torch.randn(B, 3, generator=g) * 10
    c32 = torch.randn(B, generator=g) * 3
    tok = torch.zeros(B, 768)
    tok[:, :9] = M32.reshape(B, 9)
    tok[:, 9:12] = t32
    tok[:, 12] = c32
    out = routed_model.head_pose_s(tok.to(DEV))
    P = out["pose"].double().cpu()
    conf = out["conf"].double().cpu()
    assert torch.equal(P[:, :3, 3], t32.double()), "translation"
    assert float(((conf - torch.sigmoid(c32.double())).abs() / torch.sigmoid(c32.double())).max()) <= 2.0 ** -20
    assert bool(torch.isfinite(P).all())
    R = P[:, :3, :3]
    ref = project64(M32.double())
    worst = {"exact": 0.0, "gap": 0.0}
    for i, (name, M, kind) in enumerate(cases):
        so3 = float((R[i] @ R[i].t() - torch.eye(3, dtype=torch.float64)).abs().max())
        assert so3 < 1e-5 and abs(float(torch.det(R[i])) - 1) < 1e-5, "%s: R = %s not in SO(3)" % (name, R[i].tolist())
        if kind == "exact":
            # M is a (row-)scaled rotation: R must be that rotation to fp32 rounding
            target = F.normalize(M32[i].double(), dim=-1)
            err = float((R[i] - target).abs().max())
            worst["exact"] = max(worst["exact"], err / 2.0 ** -19)
            assert err <= 2.0 ** -19, "%s: |R - M| = %.3g" % (name, err)
        elif kind == "gap":
            gap = float(ref["gap"][i])
            assert gap > 0.05, "construction: %s has gap %.3g" % (name, gap)
            bound = 2.0 * (2.0 ** -21 + 2.0 ** -18) / gap + 2.0 ** -21
            err = float((R[i] - ref["R"][i]).abs().max())
            worst["gap"] = max(worst["gap"], err / bound)
            assert err <= bound, "%s: |R - R64| = %.3g > %.3g" % (name, err, bound)
    print("pose head planted: %d cases, worst |R - M| / 2^-19 = %.4f, worst err / bound (gapped) = %.4f" % (
        B, worst["exact"], worst["gap"]), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# the 12-token golden in FP8 mode
# ---------------------------------------------------------------------------------------------------------------------

def test_pose_tokens_of_bf16_and_fp8_models_on_the_12_token_golden(cuda_model, state_dict):
    """pair_b2_48x64 (two pairs of 3 x 4 tokens): the kernel's pose from the bf16 and FP8 models' own pose tokens
    (decoder layer 12, dec_norm-ed, token 0, both views) against the float64 head on the same tokens."""
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    fp8 = STA(precision="fp8")
    fp8.load_state_dict(state_dict, strict=True)
    fp8.eval()
    g, meta, img1, img2 = golden_case("pair_b2_48x64")
    B, H, W = meta["B"], meta["H"], meta["W"]
    ts = torch.tensor([[H, W]] * B)
    toks, poses = {}, {}
    for name, m in (("bf16", cuda_model), ("fp8", fp8)):
        f1, p1 = m._encode_image(img1.cuda(), ts, normalize=False)
        f2, p2 = m._encode_image(img2.cuda(), ts, normalize=False)
        d1, d2 = m._decode_stereo(f1, f2, p1, p2, layers=(12,))
        tok = torch.cat([d1[12][:, 0, :], d2[12][:, 0, :]])
        out = m.head_pose_s(tok)
        ref = head_pose64(state_dict, tok)
        check_pose("pair_b2_48x64 %s tokens" % name, out["pose"], out["conf"], ref)
        toks[name], poses[name] = tok, (out["pose"].double(), ref)
    tok_dev = float((toks["fp8"] - toks["bf16"]).norm(dim=1).max() / toks["bf16"].norm(dim=1).max())
    pose_dev = float((poses["fp8"][0][:, :3, :3] - poses["bf16"][0][:, :3, :3]).abs().max())
    ref = poses["fp8"][1]
    print("pair_b2_48x64: fp8 vs bf16 pose tokens |d tok| / |tok| = %.3g, rotations differ by %.3g; fp8 tokens: "
          "sigma = %s, det A = %s, gap = %s" % (tok_dev, pose_dev, ref["sig"].tolist(), ref["detA"].tolist(),
                                                ref["gap"].tolist()), flush=True)
