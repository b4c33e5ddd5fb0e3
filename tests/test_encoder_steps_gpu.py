"""-m gpu: every step of the encoder's plan, run alone on designed operands, against an exact model: the conv steps
against tests/engine_model.py BIT FOR BIT, the glue steps (s2d, pool, fuse, concat, gap, finalize, heat export) against
plain fp64 references (bit for bit, except tanhf / expf: a few-ulp bound); and equivalence of the plan switches on the
real network.

Per step: one forward with keep_all on builds the plan; then the designed input (and residual / gate / second source) is
generated on the device, written with write_activation, the step runs alone with run_steps, and its output is read back.
The designed operands make both accumulator classes exact, so any lost operand piece, dropped product, mis-rounded
epilogue, wrong tap or k-block, or mis-addressed tile edge changes a checked output.  The model reads only the sampled
outputs' receptive fields from the device."""
import numpy as np
import pytest
import torch

from tests import engine_model as em

pytestmark = pytest.mark.gpu

MODES = list(em.MODES)
HALO_LAYERS = {f"s2u{u}c2" for u in range(1, 5)} | {f"s3u{u}c2" for u in range(1, 7)}
SENTINEL = 12288.0                     # exactly representable in every piece format
# forward launches of the released network with the heat-map requested: s2d, stem, pool, 39 stage 1-3 convs, 4 laterals,
# 2 x (8 top-down convs, 4 fuses, 4 output convs), heat, concat, fusion, 9 stage-4 convs, gap, mlp1, mlp2, finalize, export
FORWARD_LAUNCHES = 95


def designed_fusion_weights():
    """BiFPN fusion weights whose products and sums are exact: per output node (0.5, 0.25, 0.25) in turn."""
    fw = np.zeros((2, 20), np.float32)
    for li in range(2):
        for j in range(4):
            for i in range(3):
                fw[li, 8 + 4 * i + j] = 0.5 if i == (j + li) % 3 else 0.25
    return fw


@pytest.fixture(scope="module")
def folded():
    from dad_3dheads_b200.encoder import fold_state_dict
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    return fold_state_dict(synthetic_state_dict(0))


def _designed_encoder(folded, mode, device, seed=0, saturate=False):
    from dad_3dheads_b200.encoder import Dad3dEncoder
    layers, _ = folded
    designed, kws = em.design_network(np.random.default_rng(seed), [(n, w.shape) for n, w, _ in layers], mode, saturate)
    enc = Dad3dEncoder.from_folded(designed, designed_fusion_weights(), device, precision=mode)
    return enc, {n: (w, b) for n, w, b in designed}, kws


# ------------------------------------------------------------------------------------------------- device-side design
def t_split(x, P, fp16):
    """engine_model.split on the device (torch's bf16 conversion is RNE, its fp16 conversion RN; satfinite by clamp)."""
    r, out = x.clone(), []
    for _ in range(P):
        q = r.clamp(-65504.0, 65504.0).half().float() if fp16 else r.bfloat16().float()
        out.append(q)
        r = r - q
    return out


def t_read(x, P, fp16):
    """What read_activation returns for a tensor stored from fp32 values x: the split pieces summed smallest first."""
    ps = t_split(x, P, fp16)
    s = torch.zeros_like(x)
    for q in reversed(ps):
        s = s + q
    return s


def design_dev(shape, P, fp16, gen, k=em.K_ACT, valid_c=None, used=None):
    """engine_model.design_tensor on the device: signed 4-bit mantissas 9..15 per piece, piece p at exponent
    k - step * p (k scalar or per channel); only the first `used` pieces non-zero.  Asserts the canonical split."""
    dev = gen.device
    kk = torch.as_tensor(np.asarray(k), device=dev, dtype=torch.float32)
    used = P if used is None else used
    pieces = []
    for p in range(P):
        m = torch.randint(9, 16, shape, generator=gen, device=dev, dtype=torch.int32)
        sg = torch.randint(0, 2, shape, generator=gen, device=dev, dtype=torch.int32) * 2 - 1
        q = (m * sg).float() * torch.exp2(kk - em.PIECE_STEP[fp16] * p)
        if p >= used:
            q.zero_()
        if valid_c is not None:
            q[..., valid_c:] = 0
        pieces.append(q)
    x64 = torch.zeros(shape, dtype=torch.float64, device=dev)
    for q in reversed(pieces):
        x64 += q.double()
    x = x64.float()
    assert torch.equal(x.double(), x64)
    for a, b in zip(t_split(x, P, fp16), pieces):
        assert torch.equal(a, b), "designed values are not the canonical split"
    return x


def _shape(t):
    return (t["N"], t["H"], t["W"], t["C"])


def check_conv_steps(enc, weights, kws, mode, B, device, only=None, seed=0):
    """Run every conv step of enc's plan alone against the model; -> (plan, {step: mismatch text})."""
    P, fp16 = em.MODES[mode]
    enc.set_debug(True)
    img = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(seed)).to(device)
    enc.forward_raw(img, want_heatmap=True)
    plan = enc.describe_plan()
    gen = torch.Generator(device=device).manual_seed(seed + 1)
    bad, checked = {}, 0
    dummy_heat = torch.empty(B, 68, 64, 64, device=device)
    for i, st in enumerate(plan["steps"]):
        if st["kind"] != "conv" or (only is not None and not only(st)):
            continue
        spec = em.spec_from_step(st)
        name = st["layer"]
        w, b = weights[name]
        kw = kws[name]
        cout = w.shape[0]
        packed = em.pack(name, w, P, fp16)
        bias = np.zeros(st["n_tiles"] * st["block_n"], np.float32)
        bias[:cout] = b
        ti = st["in"]
        x = design_dev(_shape(ti), P, fp16, gen, valid_c=12 if spec.stem else None)
        if spec.stem:                                             # the s2d tensor's zero border columns
            x[:, :, :2] = 0
            x[:, :, -2:] = 0
        enc.write_activation(ti["name"], x)
        res = src2 = None
        if "res" in st:
            tr = st["res"]
            if st["res_mode"] == 4:
                k = em.K_ACT
            elif st["res_mode"] == 2:
                k = -3
            else:
                k = np.zeros(tr["C"], np.int64)
                k[:cout] = em.residual_exponent(fp16, kw)
                k[cout:] = k[0]
            r = design_dev(_shape(tr), P, fp16, gen, k=k)
            enc.write_activation(tr["name"], r)
            if st["res_mode"] == 4:
                src2 = r
            else:
                res = r
        to = st.get("out") or st["out_f32"]
        enc.write_activation(to["name"], torch.full(_shape(to), SENTINEL, device=device))
        enc.run_steps(i, 1, heatmap=dummy_heat if st["variant"] == 1 else None)
        got = enc.read_activation(to["name"])
        rows = None
        if st["rowmap_n"]:
            rows = sorted({r + d for r in st["rowmap"] for d in range(st["th"]) if r + d < spec.Ho})
        pix = em.sample_pixels(ti["N"], spec.Ho, spec.Wo, st["tw"], st["th"], st["tn"], rows=rows, seed=i)
        want = em.conv_step(spec, packed, bias, x, pix, P, fp16, res=res, src2=src2)
        checked += 1
        for sp_ in em.stored_pixels(spec, pix):
            g = em.gather(got, sp_[:, 0], sp_[:, 1], sp_[:, 2])
            if not np.array_equal(g, want):
                diff = np.argwhere(g != want)
                p0, c0 = diff[0]
                bad[f"{i}:{name}"] = (f"{len(diff)} of {g.size} differ; first at pixel {tuple(sp_[p0])} channel {c0}: "
                                      f"kernel {g[p0, c0]!r} model {want[p0, c0]!r}")
                break
        if rows is not None:                                      # rows outside the row map keep the sentinel
            untouched = [h for h in range(spec.Ho) if h not in set(rows)]
            if untouched and not bool((got[:, untouched] == SENTINEL).all()):
                bad[f"{i}:{name}:rowmap"] = "a row outside the row map was written"
        del x, res, src2, got
    assert checked > 0
    return plan, bad


def _conv_steps(plan, **kv):
    return [s for s in plan["steps"] if s["kind"] == "conv" and all(s[k] == v for k, v in kv.items())]


# batch 64 (the benchmark's batch) in the strict mode, the benchmark's default and a one-piece mode; the geometry does
# not depend on the operand format beyond what batches 2 and 5 cover in every mode
@pytest.mark.parametrize("mode,B", [(m, b) for m in MODES for b in (2, 5)] + [("fp32", 64), ("fp16x2", 64), ("bf16", 64)])
def test_conv_steps_match_model(folded, cuda_device, mode, B):
    enc, weights, kws = _designed_encoder(folded, mode, cuda_device, saturate=mode.startswith("fp16") and B == 5)
    plan, bad = check_conv_steps(enc, weights, kws, mode, B, cuda_device)
    assert not bad, bad
    P = em.MODES[mode][0]
    halo = {s["layer"] for s in _conv_steps(plan, halo=1)}
    if P == 2:
        assert HALO_LAYERS <= halo, sorted(HALO_LAYERS - halo)
    if P == 3:                                                    # one-deep rings: the 80 / 96-wide heads at three pieces
        assert {s["layer"] for s in _conv_steps(plan, stages=1)} >= {"heat", "mlp2"}
    if B == 2:                                                    # 64-wide tiles for 128-wide layers with few row tiles
        assert any(s["block_n"] == 64 and s["cout"] % 128 == 0 for s in _conv_steps(plan))
    if B == 5:                                                    # images split across tiles: tn > 1, last tile partial
        assert any(s["tn"] > 1 and s["in"]["N"] % s["tn"] for s in _conv_steps(plan))


@pytest.mark.parametrize("env,mode,B,only,expect", [
    ({"DAD3D_HALO": "0"}, "fp16x2", 5, None, lambda p: not _conv_steps(p, halo=1)),
    ({"DAD3D_TD_PARITY": "1"}, "fp16x2", 2, None, lambda p: len([s for s in _conv_steps(p) if s["parity"]]) == 16),
    ({"DAD3D_TD_PARITY": "1"}, "fp32", 2, None, lambda p: len([s for s in _conv_steps(p) if s["parity"]]) == 16),
    ({"DAD3D_HALO_CLUSTER": "2"}, "fp16x2", 64, lambda s: s["layer"].startswith("s2"),
     lambda p: {s["layer"] for s in _conv_steps(p, cl_m=2)} >= {"s2u1c2", "s2u4c2"}),
    ({"DAD3D_HALO_CLUSTER": "2"}, "bf16x2", 132, lambda s: s["layer"].startswith("s3") and s["R"] == 3,
     lambda p: {s["layer"] for s in _conv_steps(p, cl_m=2)} >= {f"s3u{u}c2" for u in range(1, 7)}),
    ({"DAD3D_HEAT_SPARSE": "0"}, "fp16x2", 5, lambda s: s["layer"] == "heat",
     lambda p: [s["variant"] for s in _conv_steps(p) if s["layer"] == "heat"] == [0]),
    ({}, "fp32", 5, lambda s: s["layer"] == "heat",
     lambda p: [s["rowmap_n"] > 0 for s in _conv_steps(p) if s["layer"] == "heat"] == [False, True]),
    ({"DAD3D_PDL": "1"}, "fp16x2", 5, None, lambda p: True),
    ({}, "fp16x2", 129, lambda s: s["layer"].startswith("mlp"),
     lambda p: all(s["tiles_w"] == 2 and s["in"]["W"] == 129 for s in _conv_steps(p) if s["layer"].startswith("mlp"))),
])
def test_conv_steps_match_model_under_switches(folded, cuda_device, monkeypatch, env, mode, B, only, expect):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    enc, weights, kws = _designed_encoder(folded, mode, cuda_device)
    plan, bad = check_conv_steps(enc, weights, kws, mode, B, cuda_device, only=only)
    assert expect(plan), "the plan does not contain the configuration this test targets"
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------ glue steps
def _ulp(x):
    return torch.from_numpy(np.spacing(np.abs(x.detach().cpu().numpy()).astype(np.float32))).to(x.device)


def check_glue_steps(enc, mode, B, device, seed=0):
    """Every non-conv step of enc's plan alone against a plain reference; -> {step: mismatch text}."""
    P, fp16 = em.MODES[mode]
    enc.set_debug(True)
    gen = torch.Generator(device=device).manual_seed(seed + 7)
    img0 = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(seed)).to(device)
    enc.forward_raw(img0, want_heatmap=True)
    plan = enc.describe_plan()
    params = torch.empty(B, 413, device=device)
    lms = torch.empty(B, 68, 2, device=device)
    heat_out = torch.empty(B, 68, 64, 64, device=device)
    bad, kinds = {}, set()

    def write(t, x):
        enc.write_activation(t["name"], x)

    def read(t):
        return enc.read_activation(t["name"])

    def exact(i, what, got, want):
        if not torch.equal(got, want):
            n = int((got != want).sum())
            bad[f"{i}:{what}"] = f"{n} of {got.numel()} values differ"

    for i, st in enumerate(plan["steps"]):
        kind = st["kind"]
        if kind == "conv":
            continue
        kinds.add(kind)
        if kind == "stem_s2d":
            img = design_dev((B, 3, 256, 256), P, fp16, gen)
            to = st["out"]
            write(to, torch.full(_shape(to), SENTINEL, device=device))
            enc.run_steps(i, 1, images=img)
            want = torch.zeros(_shape(to), device=device)
            for py in range(2):
                for px in range(2):
                    for ch in range(3):
                        want[:, :, 2:130, (py * 2 + px) * 3 + ch] = img[:, ch, py::2, px::2]
            exact(i, kind, read(to), want)
        elif kind == "stem_pool":
            ti, to = st["in"], st["out"]
            x = design_dev(_shape(ti), P, fp16, gen) if not ti["f32"] else design_dev(_shape(ti), 1, False, gen)
            write(ti, x)
            write(to, torch.full(_shape(to), SENTINEL, device=device))
            enc.run_steps(i, 1)
            want = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
            exact(i, kind, read(to), t_read(want.contiguous(), P, fp16))
        elif kind == "fuse":
            srcs, vals = [st["in"], st["in2"]] + ([st["in3"]] if "in3" in st else []), {}
            for t in srcs:                                         # a node may read one tensor twice (P7: p7td = p7x)
                if t["name"] not in vals:
                    vals[t["name"]] = design_dev(_shape(t), P, fp16, gen)
                    write(t, vals[t["name"]])
            to = st["out"]
            write(to, torch.full(_shape(to), SENTINEL, device=device))
            enc.run_steps(i, 1)
            H, W = to["H"], to["W"]
            acc = torch.zeros(_shape(to), dtype=torch.float64, device=device)
            for t, wgt in zip(srcs, st["fw"]):
                v = vals[t["name"]].double()
                sy = (torch.arange(H, device=device) * t["H"]) // H      # F.interpolate(mode="nearest")
                sx = (torch.arange(W, device=device) * t["W"]) // W
                acc += wgt * v[:, sy][:, :, sx]
            want = acc.float()
            assert torch.equal(want.double(), acc), "designed fuse is not exact"
            exact(i, kind, read(to), t_read(want, P, fp16))
        elif kind == "concat":
            tx, th, tp, to = st["in"], st["in2"], st["in3"], st["out"]
            x = design_dev(_shape(tx), P, fp16, gen)
            p5 = design_dev(_shape(tp), P, fp16, gen)
            heat = torch.randint(-64, 65, _shape(th), generator=gen, device=device).float() / 16   # [-4, 4] f32 raw
            write(tx, x), write(tp, p5), write(th, heat)
            write(to, torch.full(_shape(to), SENTINEL, device=device))
            enc.run_steps(i, 1)
            got = read(to)
            cx = tx["C"]
            exact(i, kind + ":x", got[..., :cx], x)
            exact(i, kind + ":p5", got[..., cx + 128:], p5)
            exact(i, kind + ":pad", got[..., cx + 68:cx + 128], torch.zeros_like(got[..., cx + 68:cx + 128]))
            # sigmoid(bilinear align_corners): source coordinates in fp32 as the kernel computes them, the rest in fp64
            Hh, Wh, H, W = th["H"], th["W"], to["H"], to["W"]
            fy = np.arange(H, dtype=np.float32) * (np.float32(Hh - 1) / np.float32(H - 1))
            fx = np.arange(W, dtype=np.float32) * (np.float32(Wh - 1) / np.float32(W - 1))
            y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
            y1, x1 = np.minimum(y0 + 1, Hh - 1), np.minimum(x0 + 1, Wh - 1)
            ly = torch.from_numpy((fy - y0).astype(np.float64)).to(device)[None, :, None, None]
            lx = torch.from_numpy((fx - x0).astype(np.float64)).to(device)[None, None, :, None]
            h = heat[..., :68].double()
            g = lambda ys, xs: h[:, torch.from_numpy(ys).to(device)][:, :, torch.from_numpy(xs).to(device)]  # noqa: E731
            val = (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))
            sig = 1 / (1 + torch.exp(-val))
            # fp32 evaluation of val: a few roundings of terms <= 4 (sigmoid' <= 1/4); expf + division: a few ulp
            tol = 0.25 * 8 * float(np.spacing(np.float32(4))) + 4 * _ulp(sig.float()).double()
            if P < 3:                                              # the stored pieces keep 8P / 11P bits
                tol = tol + sig.abs() * 2.0 ** -({(1, False): 8, (2, False): 16, (1, True): 11, (2, True): 22}[(P, fp16)])
            err = (got[..., cx:cx + 68].double() - sig).abs()
            if not bool((err <= tol).all()):
                bad[f"{i}:{kind}:heat"] = f"max error {float(err.max()):.3g}"
        elif kind == "gap":
            ti, to = st["in"], st["out"]
            x = design_dev(_shape(ti), P, fp16, gen, used=min(P, 2))   # 64-pixel sums of 2-piece values stay in 24 bits
            write(ti, x)
            write(to, torch.full(_shape(to), SENTINEL, device=device))
            enc.run_steps(i, 1)
            s64 = x.double().sum(dim=(1, 2)) / (ti["H"] * ti["W"])
            want = s64.float()
            assert torch.equal(want.double(), s64), "designed gap is not exact"
            exact(i, kind, read(to)[0, 0], t_read(want, P, fp16))
        elif kind == "finalize":
            ti = st["in"]
            v = torch.randint(-256, 257, _shape(ti), generator=gen, device=device).float() / 64
            write(ti, v)
            params.fill_(SENTINEL), lms.fill_(SENTINEL)
            enc.run_steps(i, 1, params=params, landmarks=lms)
            v = v[0, 0]
            exact(i, kind + ":pose", params[:, 403:], v[:, 403:413])
            exact(i, kind + ":landmarks", lms.reshape(B, 136), torch.relu(v[:, 413:549]))
            want = 3 * torch.tanh(v[:, :403].double())
            err = (params[:, :403].double() - want).abs()
            if not bool((err <= 4 * _ulp(want.float()).double()).all()):      # tanhf: 2 ulp, times 3: one rounding
                bad[f"{i}:{kind}:tanh"] = f"max error {float(err.max()):.3g}"
        elif kind == "heat_export":
            ti = st["in"]
            h = torch.randint(-64, 65, _shape(ti), generator=gen, device=device).float() / 16
            write(ti, h)
            heat_out.fill_(SENTINEL)
            enc.run_steps(i, 1, heatmap=heat_out)
            exact(i, kind, heat_out, h[..., :68].permute(0, 3, 1, 2))
    return plan, kinds, bad


@pytest.mark.parametrize("simt", [False, True])
@pytest.mark.parametrize("mode,B", [(m, 5) for m in MODES] + [("fp32", 2), ("fp16x2", 2)])
def test_glue_steps_match_model(folded, cuda_device, monkeypatch, mode, B, simt):
    if simt:
        monkeypatch.setenv("DAD3D_STEM_SIMT", "1")
    enc, _, _ = _designed_encoder(folded, mode, cuda_device)
    plan, kinds, bad = check_glue_steps(enc, mode, B, cuda_device)
    assert kinds == ({"stem_conv"} if simt else {"stem_s2d"}) | {"stem_pool", "fuse", "concat", "gap", "finalize",
                                                                 "heat_export"}
    assert not bad, bad


@pytest.mark.parametrize("mode,B", [("bf16", 2), ("fp16", 5)])
def test_stem_simt_matches_model(folded, cuda_device, monkeypatch, mode, B):
    """DAD3D_STEM_SIMT=1: fp32 FMA stem, exact on integer images and the 4-bit designed weights of a one-piece mode."""
    monkeypatch.setenv("DAD3D_STEM_SIMT", "1")
    enc, weights, _ = _designed_encoder(folded, mode, cuda_device)
    img = np.random.default_rng(5).integers(-8, 9, size=(B, 3, 256, 256)).astype(np.float32)
    enc.set_debug(True)
    x = torch.from_numpy(img).to(cuda_device)
    enc.forward_raw(torch.randn(B, 3, 256, 256, device=cuda_device))
    plan = enc.describe_plan()
    assert plan["steps"][0]["kind"] == "stem_conv"
    enc.write_activation("stem_conv", torch.full(_shape(plan["steps"][0]["out_f32"]), SENTINEL, device=cuda_device))
    enc.run_steps(0, 1, images=x)
    got = enc.read_activation("stem_conv")
    w, b = weights["stem"]
    s2d = np.zeros((B, 128, 132, 16), np.float32)
    for py in range(2):
        for px in range(2):
            s2d[:, :, 2:130, (py * 2 + px) * 3:(py * 2 + px) * 3 + 3] = img[:, :, py::2, px::2].transpose(0, 2, 3, 1)
    spec = em.ConvSpec("stem", 4, 4, pad_h=2, pad_w=0, Ho=128, Wo=128, relu=True, f32_out=True, stem=True)
    pix = em.sample_pixels(B, 128, 128, 16, 16, 1)
    packed = em.Packed([em.stem_to_4x4(w)], np.ones(64, np.float32), np.ones(64, np.float32), None)
    want = em.conv_step(spec, packed, b.astype(np.float32), s2d, pix, 1, False)
    assert np.array_equal(em.gather(got, pix[:, 0], pix[:, 1], pix[:, 2]), want)


def test_single_step_hooks_do_not_change_the_forward(folded, cuda_device):
    """The step function is shared with the forward: the launch count of a forward is the released plan's, outputs are
    bit-identical, and running all steps through run_steps is the forward."""
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.encoder import Dad3dEncoder
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    enc = Dad3dEncoder(synthetic_state_dict(0), cuda_device, precision="fp16x2")
    x = torch.randn(3, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(cuda_device)
    p0, l0, h0 = enc.forward_raw(x)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    p1, l1, h1 = enc.forward_raw(x)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == FORWARD_LAUNCHES
    n0 = _lib.launch_count()
    enc.forward_raw(x, want_heatmap=False)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == FORWARD_LAUNCHES - 1           # the support-row heat layer, no export
    assert torch.equal(p0, p1) and torch.equal(l0, l1) and torch.equal(h0, h1)
    plan = enc.describe_plan()
    p2, l2, h2 = torch.empty_like(p1), torch.empty_like(l1), torch.empty_like(h1)
    enc.run_steps(0, len(plan["steps"]), images=x, params=p2, landmarks=l2, heatmap=h2)
    assert torch.equal(p1, p2) and torch.equal(l1, l2) and torch.equal(h1, h2)
    with pytest.raises(_lib.Dad3dError):                            # workspace shared: writes would clobber
        enc.write_activation("s1u1c1", torch.zeros(3, 64, 64, 64, device=cuda_device))
    with pytest.raises(_lib.Dad3dError):
        enc.run_steps(0, len(plan["steps"]) + 1, images=x, params=p2, landmarks=l2, heatmap=h2)
    enc.set_debug(True)
    enc.forward_raw(x)
    with pytest.raises(_lib.Dad3dError):
        enc.write_activation("s1u1c1", torch.zeros(5, device=cuda_device))


# ------------------------------------------------------------------------------------------- equivalence, real network
def _run_real(monkeypatch, env, mode, x, debug=False, want_heatmap=True, names=()):
    from dad_3dheads_b200.encoder import Dad3dEncoder
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    for k in ("DAD3D_PDL", "DAD3D_HALO", "DAD3D_HALO_CLUSTER", "DAD3D_TD_PARITY", "DAD3D_HEAT_SPARSE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    enc = Dad3dEncoder(_SD(), x.device, precision=mode, want_heatmap=want_heatmap)
    if debug:
        enc.set_debug(True)
    out = enc.forward_raw(x)
    acts = {n: enc.read_activation(n) for n in names} if debug else {}
    return out, acts, enc


_sd_cache = {}


def _SD():
    if "sd" not in _sd_cache:
        from dad_3dheads_b200.encoder_weights import synthetic_state_dict
        _sd_cache["sd"] = synthetic_state_dict(0)
    return _sd_cache["sd"]


def _same(a, b):
    return all((u is None and v is None) or torch.equal(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("mode", MODES)
def test_debug_layout_is_bit_identical(monkeypatch, cuda_device, mode):
    x = torch.randn(5, 3, 256, 256, generator=torch.Generator().manual_seed(21)).to(cuda_device)
    a, _, _ = _run_real(monkeypatch, {}, mode, x, debug=True)
    b, _, _ = _run_real(monkeypatch, {}, mode, x, debug=False)
    assert _same(a, b)


@pytest.mark.parametrize("env,B", [({"DAD3D_PDL": "1"}, 5), ({"DAD3D_HALO_CLUSTER": "2"}, 64),
                                   ({"DAD3D_HALO_CLUSTER": "2"}, 132), ({"DAD3D_TD_PARITY": "1"}, 2)])
def test_switches_are_bit_identical(monkeypatch, cuda_device, env, B):
    """The switch keeps every layer's k order, so outputs and every activation both runs keep are bit-identical."""
    x = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(22)).to(cuda_device)
    a, _, enc_a = _run_real(monkeypatch, {}, "fp16x2", x, debug=True)
    b, _, enc_b = _run_real(monkeypatch, env, "fp16x2", x, debug=True)
    if "DAD3D_HALO_CLUSTER" in env:
        assert _conv_steps(enc_b.describe_plan(), cl_m=2)
    assert _same(a, b)
    names = {s["out"]["name"] for s in enc_a.describe_plan()["steps"] if s["kind"] == "conv" and "out" in s}
    names -= {n for n in names if n.endswith("_u")}             # parity launches keep the branch at half resolution
    diff = [n for n in sorted(names) if not torch.equal(enc_a.read_activation(n), enc_b.read_activation(n))]
    assert not diff, diff


@pytest.mark.parametrize("mode,env,exact", [("fp32", {}, True), ("fp16x2", {"DAD3D_HALO": "0"}, True),
                                            ("fp16x2", {}, False), ("bf16", {}, False)])
def test_sparse_heat_rows_match_full_map(monkeypatch, cuda_device, mode, env, exact):
    """Params with the sparse heat layer (want_heatmap=False) vs DAD3D_HEAT_SPARSE=0.  Bit-identical where both run the
    heat layer per tap (three pieces, or DAD3D_HALO=0); otherwise the full map runs in halo k order."""
    x = torch.randn(5, 3, 256, 256, generator=torch.Generator().manual_seed(23)).to(cuda_device)
    (pa, la, _), _, _ = _run_real(monkeypatch, env, mode, x, want_heatmap=False)
    (pb, lb, _), _, _ = _run_real(monkeypatch, dict(env, DAD3D_HEAT_SPARSE="0"), mode, x, want_heatmap=False)
    if exact:
        assert torch.equal(pa, pb) and torch.equal(la, lb)
    else:
        tol = 2e-2 if mode == "bf16" else 1e-4
        assert ((pa - pb).norm() / pb.norm()).item() < tol


@pytest.mark.parametrize("mode,B", [(m, 129) for m in MODES] + [("bf16", 512), ("fp16x2", 512)])
def test_batch_composition(monkeypatch, cuda_device, mode, B):
    """An image's outputs do not depend on the batch it runs in (the plan's tiles change with the batch)."""
    x = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(24)).to(cuda_device)
    (p, l, _), _, enc = _run_real(monkeypatch, {}, mode, x, want_heatmap=False)
    for sel in ([0], [B - 1], list(range(B - 5, B)), list(range(60, 65))):
        p1, l1, _ = enc.forward_raw(x[sel], want_heatmap=False)
        assert torch.equal(p[sel], p1) and torch.equal(l[sel], l1), (mode, B, sel)
