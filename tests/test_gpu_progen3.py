"""GPU: ProGen3 (PG_ARCH_PROGEN3) against the fp64 oracle per predicted token, under the kernel's own routing (oracle/progen3_oracle.py's
routing override), at hd 64 (d 1024, 16 heads, 4 kv heads) and hd 128 (d 2048, 16 / 4), 8 experts top-2, one expert and top_k ==
experts, gated and ungated experts, in every precision; routing agreement with the fp64 router outside a stated probability gap; MoE edge
cases (all tokens on the same experts, empty experts); bit-identical results across pass splits and runs; the goldens of the unmodified
reference (oracle/gen_golden_progen3.py) through the drop-in CLI in both checkpoint layouts."""
import ctypes as C
import io
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import progen3_oracle as O
from proteingym_b200 import _lib, checkpoint, synth
from proteingym_b200.progen3_engine import Progen3Scorer

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLDEN, "progen3_goldens.jsonl")) as _fh:
    GOLDENS = {r["name"]: r for r in map(json.loads, _fh)}
A = synth.Progen3Arch
CFGS = {
    "hd64_e8k2": A(2, 1024, 16, 4, 1024),
    "hd128_e8k2_gated": A(2, 2048, 16, 4, 1024, gated_mlp=True),
    "hd64_one_expert_gated": A(2, 1024, 16, 4, 1024, n_experts=1, top_k=1, gated_mlp=True),
    "hd64_e4k4": A(2, 1024, 16, 4, 1024, n_experts=4, top_k=4),
}
# per-token |log p - fp64 oracle| under the kernel's routing: about 4x the worst measured on an H100 80GB HBM3 at 700 W (1.98e-5,
# 6.63e-5, 1.63e-3; DESIGN.md §2)
BOUND = {"f16x3": 8e-5, "f16f8": 2.7e-4, "f16": 6.5e-3}
# a routing decision whose k-th / (k+1)-th router probabilities differ by more than this must equal the fp64 router's
GAP = {"f16x3": 1e-4, "f16f8": 1e-3, "f16": 2e-2}
LENS_FULL = (2, 63, 64, 65, 127, 128, 129, 1023, 3427)  # 3 427 = the longest ProteinGym protein (3 423) + its four added tokens
LENS = (2, 63, 64, 65, 127, 128, 129, 1023)
_CACHE = {}


def conf_state(arch, seed):
    conf = checkpoint.progen3_config(arch.config())
    return conf, checkpoint.normalise_progen3_state(conf, synth.make_progen3_state(arch, seed))


def scorer(arch, prec, seed=3, max_rows=0):
    key = (arch, prec, seed, max_rows)
    if key not in _CACHE:
        for v in _CACHE.values():
            v[0].close()
        _CACHE.clear()  # one model on the device at a time
        conf, st = conf_state(arch, seed)
        _CACHE[key] = (Progen3Scorer(conf, st, precision=prec, max_rows=max_rows), conf, st)
    return _CACHE[key]


def token_rows(lens, seed):
    rng = np.random.default_rng(seed)
    return [[1] + list(rng.integers(6, 34, n - 1)) for n in sorted(lens)]


def routing(sc, layer, k, cap):
    """(experts, weights) of every token row of the last pass (at most ``cap`` rows), [rows, k] each."""
    n = C.c_int32()
    e = torch.empty(cap * k, dtype=torch.int32, device=sc.device)
    w = torch.empty(cap * k, dtype=torch.float32, device=sc.device)
    _lib.check(sc.lib.pg_progen3_routing(sc.handle, layer, e.data_ptr(), w.data_ptr(), C.byref(n), sc.stream()), sc.handle)
    torch.cuda.synchronize()
    return e[:n.value * k].view(-1, k).cpu().numpy(), w[:n.value * k].view(-1, k).cpu().numpy()


def run_rows(sc, conf, rows):
    """Kernel per-token log-probs per row and the kernel's routing per row and layer (rows sorted by length: one batch, one pass)."""
    _, lp_rows = sc.token_sums(rows, return_rows=True)
    T = len(rows[-1])
    per_layer = [routing(sc, l, conf.top_k, len(rows) * T) for l in range(conf.layers)]
    out = []
    for b, r in enumerate(rows):
        tok = lp_rows[b][np.arange(len(r) - 1), np.asarray(r[1:])]
        rt = [(e[b * T:b * T + len(r)], w[b * T:b * T + len(r)]) for e, w in per_layer]
        out.append((tok, rt))
    return out


def check_against_oracle(arch, prec, lens, seed=3):
    sc, conf, st = scorer(arch, prec, seed)
    rows = token_rows(lens, seed)
    worst, flips, inside, min_gap, decisions = 0.0, 0, 0, np.inf, 0
    for r, (tok, rt) in zip(rows, run_rows(sc, conf, rows)):
        want, routes = O.token_logp(st, conf, r, torch.float64, routing=rt)
        err = np.abs(tok.astype(np.float64) - want)
        assert np.isfinite(tok).all()
        worst = max(worst, float(err.max()))
        for (ke, _), (_, _, probs) in zip(rt, routes):
            gaps = O.topk_gaps(probs, conf.top_k)
            own = np.sort(np.argsort(-probs, axis=1, kind="stable")[:, :conf.top_k], axis=1)
            agree = (np.sort(ke, axis=1) == own).all(axis=1)
            decisions += len(gaps)
            inside += int((gaps <= GAP[prec]).sum())
            min_gap = min(min_gap, float(gaps.min()))
            flips += int((~agree).sum())
            assert agree[gaps > GAP[prec]].all(), f"routing differs from the fp64 router at a gap above {GAP[prec]}"
    print(f"\n{arch} {prec}: worst |dlogp| {worst:.3e}; {decisions} routing decisions, {inside} within gap {GAP[prec]}, "
          f"{flips} differing from fp64, smallest gap {min_gap:.3e}")
    assert worst < BOUND[prec], worst


@pytest.mark.parametrize("prec", ["f16x3", "f16f8", "f16"])
def test_hd64_e8k2_per_token_vs_fp64(prec):
    check_against_oracle(CFGS["hd64_e8k2"], prec, LENS_FULL)


@pytest.mark.parametrize("prec", ["f16x3", "f16f8", "f16"])
def test_hd128_gated_per_token_vs_fp64(prec):
    check_against_oracle(CFGS["hd128_e8k2_gated"], prec, LENS)


@pytest.mark.parametrize("name", ["hd64_one_expert_gated", "hd64_e4k4"])
def test_special_expert_counts_vs_fp64(name):
    check_against_oracle(CFGS[name], "f16f8", LENS)


def test_all_tokens_on_the_same_experts():
    """A zero router: every probability is exactly 1/E, so every token takes the experts torch.topk's CPU tie order picks (6 and 5 of 8),
    the other experts stay empty, and the segments are not multiples of 128 rows."""
    arch = A(2, 1024, 16, 4, 1024, n_experts=8, top_k=2)
    conf, st = conf_state(arch, 4)
    for l in range(arch.layers):
        st[f"layers.{l}.block_sparse_moe.gate.weight"] = torch.zeros_like(st[f"layers.{l}.block_sparse_moe.gate.weight"])
    want_e = torch.topk(torch.full((1, 8), 0.125), 2, dim=-1).indices[0].numpy()
    sc = Progen3Scorer(conf, st, precision="f16x3")
    try:
        rows = token_rows((3, 77, 200), 4)
        for r, (tok, rt) in zip(rows, run_rows(sc, conf, rows)):
            for e, w in rt:
                assert (e == want_e).all() and (w == 0.5).all()
            want, _ = O.token_logp(st, conf, r, torch.float64, routing=rt)
            assert np.abs(tok - want).max() < BOUND["f16x3"]
    finally:
        sc.close()


@pytest.mark.parametrize("E,k", [(8, 2), (6, 4), (16, 3), (64, 1), (64, 8)])
def test_router_ties_follow_torch_topk(E, k):
    """Duplicated router rows give exactly equal probabilities; the kernel's selection and order must be torch.topk's on the CPU wherever
    the distinct probabilities are further apart than the f16x3 gap bound."""
    arch = A(2, 1024, 16, 4, 256, n_experts=E, top_k=k)
    conf, st = conf_state(arch, 6)
    rng = np.random.default_rng(E * 10 + k)
    for l in range(arch.layers):
        g = st[f"layers.{l}.block_sparse_moe.gate.weight"]
        st[f"layers.{l}.block_sparse_moe.gate.weight"] = g[torch.as_tensor(rng.integers(0, max(2, E // 3), E))].clone()
    sc = Progen3Scorer(conf, st, precision="f16x3")
    checked = 0
    try:
        rows = token_rows((64, 200), 5)
        for r, (tok, rt) in zip(rows, run_rows(sc, conf, rows)):
            _, routes = O.token_logp(st, conf, r, torch.float64, routing=rt)
            for (ke, _), (_, _, probs) in zip(rt, routes):
                for t in range(len(r)):
                    u = np.unique(probs[t])
                    if len(u) > 1 and np.diff(u).min() <= GAP["f16x3"]:
                        continue
                    want = torch.topk(torch.tensor(probs[t:t + 1], dtype=torch.float32), k, dim=-1).indices[0].numpy()
                    assert (ke[t] == want).all(), (t, ke[t], want, probs[t])
                    checked += 1
    finally:
        sc.close()
    print(f"\nE {E} top-{k}: {checked} tied routing decisions equal torch.topk's")
    assert checked > 0


def test_bit_identical_across_pass_splits_and_runs():
    arch = CFGS["hd64_e8k2"]
    rows = token_rows((5, 70, 130, 130, 300, 301), 9)
    sc, conf, st = scorer(arch, "f16f8", 3)
    a = sc.token_sums(rows)
    b = sc.token_sums(rows)
    sc_small, _, _ = scorer(arch, "f16f8", 3, max_rows=700)  # two or more passes per batch
    c = sc_small.token_sums(rows)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_goldens_through_the_cli(tmp_path):
    from proteingym_b200 import score_progen3
    worst = 0.0
    for i, (name, g) in enumerate(GOLDENS.items()):
        arch = A(**g["arch"])
        folder = tmp_path / name
        synth.write_progen3_checkpoint(str(folder), arch, g["seed"], layout="megablocks" if i % 2 and arch.n_experts > 1 else "eager")
        fasta = tmp_path / f"{name}.fasta"
        fasta.write_text("".join(f">{k} some description\n{v[:40]}\n{v[40:]}\n" for k, v in g["records"].items()))
        out = tmp_path / f"{name}.csv"
        args = score_progen3.create_parser().parse_args(["--model-name", str(folder), "--fasta-path", str(fasta), "--output-path", str(out)])
        if "error" in g:  # the reference fails (top_k == experts): the scorer weights each expert by its own renormalised weight
            assert "einsum" in g["error"]
            df = score_progen3.main(args)
            conf, st = conf_state(arch, g["seed"])
            ll, _ = O.score(st, conf, [g["records"][k] for k in sorted(g["records"])])
            assert np.abs(df["log_likelihood"].to_numpy() - ll).max() < 1e-3
            continue
        score_progen3.main(args)
        got, want = pd.read_csv(out), pd.read_csv(io.StringIO(g["csv"]))
        assert list(got.columns) == list(want.columns) and list(got["sequence_id"]) == list(want["sequence_id"])
        err = np.abs(got["log_likelihood"].to_numpy() - want["log_likelihood"].to_numpy()).max()
        rel = np.abs(got["perplexity"].to_numpy() / want["perplexity"].to_numpy() - 1).max()
        print(f"\ngolden {name}: max |ll - reference| {err:.2e}, max perplexity rel. error {rel:.2e}")
        worst = max(worst, err)
        assert err < 1e-3 and rel < 1e-3
    print(f"\ngoldens: worst |ll - reference| {worst:.2e}")
