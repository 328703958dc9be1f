"""Simulated Byzantine clients on the GPU: K22 against the CPU oracle (odd P, misaligned and padded arenas, C up to 256, the
mask, h = 0 / 1 / many, a ResNet-18-sized row), its determinism and its binding's checks; the fused round kernel's
sign_flip / gaussian phase against the oracle over every warps-per-pair setting and cluster size and with the aggregation
rules, compression and the defense; the fused kernel against the generic executor, CUDA-graph replay, routing, and launches
without an attack against a fixture recorded before the attack phase existed."""
import copy
import os

import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from test_gpu_small_round import make_state, to_cuda
from test_robust_agg import _same

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fused_no_attack.pt")   # the launches of golden_states


def _arena(C, M, P, pad=0, misaligned=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(M, P + pad, generator=g)
    rows = theta[None, :, :P] + torch.randn(C, M, P, generator=g) * (1.0 + (torch.arange(C, dtype=torch.float32) % 7)[:, None, None])
    n = (torch.rand(C, M, generator=g) * 3).floor()
    n[:, 0] = 0
    n[0, 0] = 2                                            # slot 0: only client 0 (an attacker) trained: h = 0
    if M > 1:
        n[:, 1] = 0
        n[[0, 1], 1] = 1                                   # slot 1: h = 1
    return theta, rows, n


def _gpu_rows(rows, misaligned):
    if not misaligned:
        return rows.cuda()
    buf = torch.empty(rows.numel() + 1, device="cuda")
    out = buf[1:].view(rows.shape)                         # 4-byte aligned only: the scalar path
    out.copy_(rows)
    return out


CASES = [dict(C=9, M=4, P=13), dict(C=9, M=3, P=64, pad=5), dict(C=16, M=3, P=1001, misaligned=True),
         dict(C=256, M=2, P=517, pad=3), dict(C=7, M=3, P=4096, masked=True), dict(C=5, M=2, P=2048, misaligned=True, masked=True)]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", ["sign_flip", "alie", "ipm", "gaussian"])
def test_k22_matches_oracle(case, kind):
    C, M, P = case["C"], case["M"], case["P"]
    theta, rows, n = _arena(C, M, P, case.get("pad", 0), seed=C + P)
    att = ref.attacker_clients(C, max(1, C // 4), 5)
    att[0] = True
    mask = (torch.arange(P) % 7 != 3) if case.get("masked") else None
    seed = ref.attack_seed(11, 3)
    want = rows.clone()
    ref.attack_slots_(want, theta, n, att, kind, 1.75, mask, seed)
    got = _gpu_rows(rows, case.get("misaligned", False))
    ops.attack_slots_(got, theta.cuda(), n.cuda(), att.cuda(), kind, 1.75, None if mask is None else mask.cuda(), seed)
    torch.cuda.synchronize()
    if kind == "gaussian":   # fp32 sqrtf / logf / cospif on the device against the float64 host noise, as weak DP
        assert torch.allclose(got.cpu(), want, rtol=1e-5, atol=1e-5), (got.cpu() - want).abs().max()
    else:
        assert _same(got.cpu(), want), (got.cpu() - want).abs().max()
    assert not torch.equal(want, rows)


@pytest.mark.parametrize("kind", ["sign_flip", "alie", "ipm"])
def test_k22_resnet18_sized_row(kind):
    C, M, P = 4, 1, 11 * (1 << 20) + 3
    g = torch.Generator().manual_seed(2)
    theta = torch.randn(M, P, generator=g)
    rows = theta[None] + torch.randn(C, M, P, generator=g)
    n = torch.ones(C, M)
    att = torch.tensor([False, True, False, True])
    want = rows.clone()
    ref.attack_slots_(want, theta, n, att, kind, 0.5)
    got = rows.cuda()
    ops.attack_slots_(got, theta.cuda(), n.cuda(), att.cuda(), kind, 0.5)
    torch.cuda.synchronize()
    assert _same(got.cpu(), want)


@pytest.mark.parametrize("kind", ["sign_flip", "gaussian", "alie", "ipm"])
def test_k22_is_bit_identical_across_launches(kind):
    theta, rows, n = _arena(64, 3, 3001, seed=4)
    att = ref.attacker_clients(64, 20, 1).cuda()
    a, b = rows.cuda(), rows.cuda()
    for x in (a, b):
        ops.attack_slots_(x, theta.cuda(), n.cuda(), att, kind, 3.0, None, 99)
    torch.cuda.synchronize()
    assert _same(a, b)


def test_k22_binding_rejects_bad_arguments():
    from feddrift_b200.ops import _ext
    ext = _ext.load(required=True)
    rows, th, n = torch.zeros(3, 2, 5, device="cuda"), torch.zeros(2, 5, device="cuda"), torch.ones(3, 2, device="cuda")
    att = torch.ones(3, dtype=torch.uint8, device="cuda")
    ext.attack_slots(rows, th, n, att, 1, 1.0, None, 0)
    bad = [
        (rows.double(), th, n, att, 1, 1.0), (rows, th.double(), n, att, 1, 1.0), (rows, th, n.double(), att, 1, 1.0),
        (rows, th, n, att.bool(), 1, 1.0), (rows, th, n, att.int(), 1, 1.0),
        (rows, th, n, torch.ones(4, dtype=torch.uint8, device="cuda"), 1, 1.0),
        (rows, th, n, torch.ones(2, dtype=torch.uint8, device="cuda"), 1, 1.0),
        (rows, torch.zeros(3, 5, device="cuda"), n, att, 1, 1.0), (rows, torch.zeros(2, 4, device="cuda"), n, att, 1, 1.0),
        (rows, th, torch.ones(2, 2, device="cuda"), att, 1, 1.0), (rows.transpose(0, 1), th, n, att, 1, 1.0),
        (rows, th, n, att, 0, 1.0), (rows, th, n, att, 5, 1.0), (rows, th, n, att, 1, 0.0), (rows, th, n, att, 1, -1.0),
        (rows, th, n, att, 1, float("inf")), (rows, th, n, att, 1, float("nan")), (rows, th, n, att, 1, 1e39),
    ]
    for args in bad:
        with pytest.raises(RuntimeError):
            ext.attack_slots(*args, None, 0)
    with pytest.raises(RuntimeError):
        ext.attack_slots(rows, th, n, att, 1, 1.0, torch.ones(4, dtype=torch.uint8, device="cuda"), 0)
    with pytest.raises(RuntimeError):
        ext.attack_slots(rows, th, n, att, 1, 1.0, None, -1)
    with pytest.raises(ValueError):
        ops.attack_slots_(rows, th, n, att, "label_flip", 1.0)


# ----------------------------------------------------------------------------- fused round kernel
def _atk(st, kind="sign_flip", a=3, s=2.0):
    C = st["X"].shape[1]
    return dict(st, attack_type=kind, attack_clients=a, attack_scale=s, attackers=ref.attacker_clients(C, a, 7))


SHAPES = [dict(), dict(kind="lr", hid=0), dict(din=2, hid=4), dict(kind="fnn", din=4, hid=8, dout=3), dict(C=37, M=4)]


def _uploads_match(st, kind):
    """One launch with client_out, with and without the attack from the same state: the attacked uploads are K22's (and the
    oracle's) poisoning of the honest ones."""
    C, M, P = st["X"].shape[1], *st["theta"].shape
    plain = to_cuda(copy.deepcopy({k: v for k, v in st.items() if not k.startswith("attack")}))
    plain["client_out"] = torch.zeros(C, M, P, device="cuda")
    g = to_cuda(copy.deepcopy(st))
    g["client_out"] = torch.zeros(C, M, P, device="cuda")
    theta0 = g["theta"].clone()
    ops.fed_round_small(plain, 1)
    ops.fed_round_small(g, 1)
    torch.cuda.synchronize()
    up = plain["client_out"]
    sel = (up != 0).any(-1).float()
    want = up.clone()
    ops.attack_slots_(want, theta0, sel, st["attackers"].cuda(), kind, st["attack_scale"], None,
                      ref.attack_seed(st["seed"], int(st["round0"])))
    if kind == "gaussian":
        assert torch.allclose(g["client_out"], want, rtol=1e-5, atol=1e-5)
    else:
        assert _same(g["client_out"], want)
        cpu = up.cpu().clone()
        ref.attack_slots_(cpu, theta0.cpu(), sel.cpu(), st["attackers"], kind, st["attack_scale"])
        assert _same(g["client_out"].cpu(), cpu)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("wpp", [1, 2, 4])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", ["sign_flip", "gaussian"])
def test_fused_phase_matches_oracle(shape, wpp, G, kind):
    st = dict(_atk(make_state(**shape), kind), cluster=G, warps_per_pair=wpp)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)
    ref.fed_round_small(st, 3)
    torch.cuda.synchronize()
    assert torch.allclose(g["theta"].cpu(), st["theta"], rtol=1e-4, atol=1e-5), (g["theta"].cpu() - st["theta"]).abs().max()
    _uploads_match(st, kind)


COMBOS = [dict(aggregation_rule="median"), dict(aggregation_rule="multi_krum", krum_f=1, krum_m=2),
          dict(compression="qsgd", quantize_level=4, quantize_bucket=8), dict(compression="eftopk", topk_ratio=0.3),
          dict(defense="norm_diff_clipping", norm_bound=0.5),
          dict(aggregation_rule="median", compression="eftopk", topk_ratio=0.3, defense="norm_diff_clipping", norm_bound=0.5)]


@pytest.mark.parametrize("combo", COMBOS)
@pytest.mark.parametrize("kind", ["sign_flip", "gaussian"])
def test_fused_phase_with_rules_compression_and_defense(combo, kind):
    st = dict(_atk(make_state(C=12), kind), cluster=4, **combo)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)
    ref.fed_round_small(st, 3)
    torch.cuda.synchronize()
    assert torch.allclose(g["theta"].cpu(), st["theta"], rtol=1e-4, atol=1e-5), (g["theta"].cpu() - st["theta"]).abs().max()
    if "compression" not in combo:   # eftopk's residual and QSGD's draws are checked by the oracle comparison above
        _uploads_match(st, kind)


def test_fused_no_attack_is_bit_identical_to_the_kernel_without_an_attack_phase():
    """The fixture holds the fused kernel's results of these launches (no attack configured) recorded on an H100 with the
    kernel as it was before the attack phase was added."""
    gold = torch.load(GOLDEN)
    for name, st in golden_states().items():
        g = to_cuda(st)
        out = ops.fed_round_small(g, 3)
        torch.cuda.synchronize()
        assert _same(g["theta"].cpu(), gold[name]["theta"]), name
        assert _same(out["metrics"].cpu(), gold[name]["metrics"]), name


def golden_states():
    base = make_state(C=12)
    return {
        "mean": dict(copy.deepcopy(base), cluster=4),
        "median_qsgd": dict(copy.deepcopy(base), cluster=2, aggregation_rule="median", compression="qsgd", quantize_level=4,
                            quantize_bucket=8),
        "krum_eftopk_clip": dict(copy.deepcopy(base), cluster=4, aggregation_rule="multi_krum", krum_f=1, krum_m=2,
                                 compression="eftopk", topk_ratio=0.3, defense="norm_diff_clipping", norm_bound=0.5),
        "lr_wpp2": dict(make_state(kind="lr", hid=0), warps_per_pair=2),
    }


def test_honest_attackers_mask_changes_nothing():
    """An attack whose only attacker never trains takes the kAttack kernel and leaves every upload as trained."""
    st = make_state(C=12)
    st["participation"] = torch.ones(3, 12, dtype=torch.bool)
    st["participation"][:, 5] = False
    att = torch.zeros(12, dtype=torch.bool)
    att[5] = True
    a = to_cuda(dict(copy.deepcopy(st), attack_type="sign_flip", attack_clients=1, attackers=att, cluster=4))
    b = to_cuda(dict(copy.deepcopy(st), cluster=4))
    ops.fed_round_small(a, 3)
    ops.fed_round_small(b, 3)
    torch.cuda.synchronize()
    assert _same(a["theta"], b["theta"]) and _same(a["opt_m"], b["opt_m"])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, attack_type="sign_flip", attack_clients=3, attack_scale=3.0)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


@pytest.mark.parametrize("kind", ["sign_flip", "gaussian", "alie", "ipm"])
def test_fused_and_generic_agree_on_a_small_cfg2_like_run(kind):
    kw = dict(client_num_in_total=20, sample_num=60, comm_round=3, total_train_iteration=2, attack_type=kind, attack_clients=4)
    a, b = _sim(**kw), _sim(**kw)
    b.algo.fused_ok = lambda: False
    a.run()
    b.run()
    from feddrift_b200.ops import small_round
    assert a._use_fused() == (kind in ("sign_flip", "gaussian")) and small_round.LAUNCH_COUNT["fed_round_small"] > 0
    assert torch.allclose(a.bank.theta, b.bank.theta, rtol=1e-4, atol=1e-4), (a.bank.theta - b.bank.theta).abs().max()
    assert abs(a.history[-1]["test_acc_honest"] - b.history[-1]["test_acc_honest"]) < 0.02


def test_round_graph_replay_matches_non_graph_path():
    def make():
        sim = _sim(client_num_per_round=5, attack_type="gaussian", attack_scale=0.2)
        sim.run_time_step(0, rounds=3)
        sim.begin_time_step(1)
        sim.run_rounds(1)
        sim.args.rounds_per_launch = 1
        return sim

    a, b = make(), make()
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss", "test_acc_honest"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert _same(a.bank.theta, b.bank.theta)


def test_fits_routes_alie_and_ipm_to_the_generic_executor_and_cfg2_runs_fused():
    from feddrift_b200.experiments.configs import CONFIGS
    from feddrift_b200.ops import small_round
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    for atk in (None, "none", "sign_flip", "gaussian"):
        assert small_round.fits("fnn", 4, 8, 3, 100, 2, 0, attack=atk)
    for atk in ("alie", "ipm"):
        assert not small_round.fits("fnn", 4, 8, 3, 100, 2, 0, attack=atk)
    for kind, fused in (("sign_flip", True), ("alie", False), ("ipm", False)):
        cfg = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"], attack_type=kind, attack_clients=20, comm_round=2,
                   total_train_iteration=2)
        s = DriftSim(make_args(**cfg), device="cuda", sink=MetricsSink())
        s.begin_time_step(0)
        assert s._use_fused() == fused
        n0 = small_round.LAUNCH_COUNT["fed_round_small"]
        s.run_rounds(2)
        assert (small_round.LAUNCH_COUNT["fed_round_small"] > n0) == fused and torch.isfinite(s.bank.theta).all()
    with pytest.raises(RuntimeError):   # the kernel refuses ALIE / IPM instead of running them unattacked
        st = to_cuda(_atk(make_state(), "sign_flip"))
        st["_native"] = {}
        small_round.run_native(dict(st, attack_type="alie"), 1)
