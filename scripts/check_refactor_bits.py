"""Outputs of every model family on seeded synthetic models, in one .npz: run it on two builds of the library and compare the files
with --compare. A change that only moves device code between files must leave every array np.array_equal.

    python scripts/check_refactor_bits.py out.npz
    python scripts/check_refactor_bits.py --compare a.npz b.npz

ESM-1v scores in f16x3 / f16f8 / f16d / f16, an ESM2 of the 35M release's shape (480 wide, 24-wide heads: the padded LayerNorm) in
f16f8, Tranception mutant scores with and without prefix reuse and rows with a three-way retrieval fusion in f16x3 / f16f8, a
two-layer MSA Transformer table (a full and a pruned last layer) in f16x3 / f16f8, and RITA, ProGen2 and ProtGPT2 scores of a 900-residue
wild type's substitutions and indels with and without prefix reuse in f16f8. Every run with prefix reuse also records its token-row
counts (reuse_rows). The load paths the runs above leave out have a run each (loads()): ESM C in f16f8 / f16x3, an ESM-1b with
emb_layer_norm_before, an MSA Transformer without msa_position_embedding, ProGen2 with 80-wide heads (128-wide slots), RITA with an
untied head, and PoET with and without its final norm in f16x3 / f16f8 (per-token log p and layer 0 of the context record). Runs split
into several passes have a run each (passes()): ProGen3 in f16x3 / f16f8, PoET's per-sequence sums, and ESM-1v wt-marginals over
overlapping 1024-token windows (pg_forward_logprobs). Every array <name> comes with <name>.launches: the library's launch count
(pg_launch_count) over the work since the array stored before it."""
import os
import sys

import numpy as np


class Runs(dict):
    """Arrays by name; storing <name> also stores <name>.launches, the launches counted since the previous store."""

    def __init__(self):
        super().__init__()
        from proteingym_b200 import _lib
        self.lib = _lib.load()
        self.mark = self.lib.pg_launch_count()

    def __setitem__(self, name, value):
        n = self.lib.pg_launch_count()
        super().__setitem__(name, value)
        super().__setitem__(name + ".launches", np.array([n - self.mark], dtype=np.int64))
        self.mark = n


def collect():
    import pandas as pd
    from proteingym_b200 import checkpoint, msa_engine, synth
    from proteingym_b200.esm_engine import EsmScorer
    from proteingym_b200.tranception_engine import TranceptionScorer
    out = Runs()
    seq = synth.random_protein(200, 3)
    muts = synth.sample_mutants(seq, 400, 4, multi_frac=0.2)
    for name, arch, modes in (("esm1v", synth.EsmArch("esm1v", 3, 256, 4, 1024), ("f16x3", "f16f8", "f16d", "f16")),
                              ("esm2_35m", synth.EsmArch("esm2", 2, 480, 20, 1920), ("f16f8",))):
        st = checkpoint.normalise_synth_state(arch, synth.make_esm_state(arch, seed=1))
        for mode in modes:
            sc = EsmScorer(checkpoint.config_from_synth(arch), st, precision=mode)
            out[f"{name}.{mode}"] = np.asarray(sc.score_assay(seq, muts))
            sc.close()
    arch = synth.TranceptionArch(2, 768, 12, 3072)
    cfg = {"n_embd": 768, "n_head": 12, "n_layer": 2, "n_ctx": 1024, "n_inner": 3072, "vocab_size": 25, "layer_norm_epsilon": 1e-5,
           "activation_function": "squared_relu"}
    st = {k[len("transformer."):]: v for k, v in synth.make_tranception_state(arch, 5).items() if k.startswith("transformer.")}
    wt = synth.random_protein(400, 6)
    m = synth.sample_mutants(wt, 120, 7)
    dms = pd.DataFrame({"mutant": m, "mutated_sequence": [synth.apply_mutant(wt, x) for x in m]})
    L = 300
    rng = np.random.RandomState(8)
    prior = np.log(rng.dirichlet(np.ones(25), size=L)).astype(np.float32)
    prior2 = np.log(rng.dirichlet(np.ones(25), size=L)).astype(np.float32)
    for mode in ("f16x3", "f16f8"):
        for reuse in (True, False):
            sc = TranceptionScorer(cfg, st, precision=mode)
            sc.prefix_reuse = reuse
            df = sc.score_mutants(dms, wt)
            out[f"tranception.{mode}.reuse{int(reuse)}"] = df.select_dtypes("number").to_numpy()
            out[f"tranception.{mode}.reuse{int(reuse)}.rows"] = np.asarray(sc.reuse_rows)
            sc.close()
        sc = TranceptionScorer(cfg, st, precision=mode)
        sums, rows = sc.sequence_logprobs([wt[:L]], prior=prior, windows=[(0, L)], alpha=0.6, msa_start=40, msa_end=L - 30, prior2=prior2,
                                          beta=0.3, first_col=5, return_rows=True)
        out[f"tranception.{mode}.fusion3"] = rows[0]
        out[f"tranception.{mode}.fusion3.sum"] = sums
        sc.close()
    arch = synth.MsaArch(2, 256, 4, 1024)
    cfg = checkpoint.config_from_msa_synth(arch)
    st = checkpoint.normalise_msa_synth_state(arch, synth.make_msa_state(arch, 9))
    toks = msa_engine.tokenize_alignment(synth.random_alignment(synth.random_protein(90, 10), 24, seed=11))
    R, Cc = toks.shape
    pos = np.arange(1, Cc, 7).astype(np.int32)
    for mode in ("f16x3", "f16f8"):
        sc = msa_engine.MsaScorer(cfg, st, precision=mode, max_rows=msa_engine.default_max_rows(cfg, R, Cc, want=4))
        out[f"msa.{mode}"] = sc.masked_marginal_rows(toks, pos).cpu().numpy()
        sc.close()
    out.update(decoders())
    out.update(loads())
    out.update(passes())
    return out


def decoders():
    """RITA, ProGen2 and ProtGPT2 on seeded two-layer models: score() of substitutions (first change before and after token 128) and
    indels of one wild type, with prefix reuse on and off."""
    from proteingym_b200 import checkpoint, synth
    from proteingym_b200.progen2_engine import Progen2Scorer
    from proteingym_b200.protgpt2_engine import Protgpt2Scorer, Protgpt2Tokenizer
    from proteingym_b200.rita_engine import RitaScorer, RitaTokenizer
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
    wt = synth.random_protein(900, 12)
    prots = [synth.apply_mutant(wt, m) for m in synth.sample_mutants(wt, 48, 13, multi_frac=0.25)] + synth.random_indels(wt, 16, 14)

    def rita():
        arch = synth.RitaArch(2, 256, 4)
        st = synth.make_rita_state(arch, 15)
        ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()
              if "inv_freq" not in k and k != "lm_head.weight"}
        conf = checkpoint.RitaConfig(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, True)
        return RitaScorer(conf, ws, st["transformer.layers.0.self_attention.rotary_embedding.inv_freq"],
                          RitaTokenizer(os.path.join(golden, "rita_tokenizer_plain")), precision="f16f8")

    def progen2():
        a = synth.Progen2Arch(2, 512, 8, 32)
        st = synth.make_progen2_state(a, 16, buffers=False)
        ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()}
        return Progen2Scorer(checkpoint.Progen2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.rotary_dim, a.n_positions), ws,
                             precision="f16f8")

    def protgpt2():
        a = synth.Protgpt2Arch(2, 256, 4)
        st = synth.make_protgpt2_state(a, 17)
        ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items() if k != "lm_head.weight"}
        return Protgpt2Scorer(checkpoint.Protgpt2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.n_positions), ws,
                              Protgpt2Tokenizer(os.path.join(golden, "protgpt2_tokenizer")), precision="f16f8")
    out = Runs()
    for name, make in (("rita", rita), ("progen2", progen2), ("protgpt2", protgpt2)):
        sc = make()
        for reuse in (True, False):
            sc.prefix_reuse = reuse
            sc.reuse_rows = [0, 0]
            out[f"{name}.f16f8.reuse{int(reuse)}"] = sc.score(prots, wt=wt)
            out[f"{name}.f16f8.reuse{int(reuse)}.rows"] = np.asarray(sc.reuse_rows)
        sc.close()
    return out


def loads():
    """One run per weight-load path that collect() and decoders() do not reach."""
    from proteingym_b200 import checkpoint, msa_engine, synth
    from proteingym_b200 import poet_engine as E
    from proteingym_b200.esm_engine import EsmScorer
    from proteingym_b200.progen2_engine import Progen2Scorer
    from proteingym_b200.rita_engine import RitaScorer, RitaTokenizer
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
    out = Runs()
    seq = synth.random_protein(150, 21)
    muts = synth.sample_mutants(seq, 200, 22, multi_frac=0.2)
    st = synth.make_esmc_state(synth.EsmcArch(2, 256, 512), seed=23)
    for mode in ("f16f8", "f16x3"):
        sc = EsmScorer(checkpoint.esmc_config_from_state(st), st, precision=mode)
        out[f"esmc.{mode}"] = np.asarray(sc.score_assay(seq, muts))
        sc.close()
    arch = synth.EsmArch("esm1v", 2, 256, 4, 1024, emb_layer_norm_before=True)
    sc = EsmScorer(checkpoint.config_from_synth(arch), checkpoint.normalise_synth_state(arch, synth.make_esm_state(arch, seed=24)),
                   precision="f16f8")
    out["esm1b_ln_before.f16f8"] = np.asarray(sc.score_assay(seq, muts))
    sc.close()
    arch = synth.MsaArch(2, 256, 4, 1024, embed_positions_msa=False)
    cfg = checkpoint.config_from_msa_synth(arch)
    st = checkpoint.normalise_msa_synth_state(arch, synth.make_msa_state(arch, 25))
    toks = msa_engine.tokenize_alignment(synth.random_alignment(synth.random_protein(90, 26), 24, seed=27))
    R, Cc = toks.shape
    sc = msa_engine.MsaScorer(cfg, st, precision="f16f8", max_rows=msa_engine.default_max_rows(cfg, R, Cc, want=4))
    out["msa_no_row_pos.f16f8"] = sc.masked_marginal_rows(toks, np.arange(1, Cc, 7).astype(np.int32)).cpu().numpy()
    sc.close()
    wt = synth.random_protein(300, 28)
    prots = [synth.apply_mutant(wt, m) for m in synth.sample_mutants(wt, 24, 29)] + synth.random_indels(wt, 8, 30)
    a = synth.Progen2Arch(2, 640, 8, 32)
    st = synth.make_progen2_state(a, 31, buffers=False)
    ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()}
    sc = Progen2Scorer(checkpoint.Progen2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.rotary_dim, a.n_positions), ws,
                       precision="f16f8")
    out["progen2_hd80.f16f8"] = sc.score(prots, wt=wt)
    sc.close()
    arch = synth.RitaArch(2, 256, 4)
    st = synth.make_rita_state(arch, 32, untied=True)
    ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items() if "inv_freq" not in k}
    sc = RitaScorer(checkpoint.RitaConfig(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, False), ws,
                    st["transformer.layers.0.self_attention.rotary_embedding.inv_freq"],
                    RitaTokenizer(os.path.join(golden, "rita_tokenizer_plain")), precision="f16f8")
    out["rita_untied.f16f8"] = sc.score(prots, wt=wt)
    sc.close()
    rng = np.random.default_rng(33)

    def row(n):
        return np.concatenate([[E.START], rng.integers(0, 20, size=n - 2), [E.STOP]]).astype(np.int64)
    ctx = [row(n) for n in (40, 130, 7, 90)]
    variants = [row(n) for n in (20, 65, 128, 129)]
    for norm in (False, True):
        arch = synth.PoetArch(2, 256, 4, norm=norm)
        st = synth.make_poet_state(arch, seed=34)
        conf = checkpoint.PoetConfig(arch.layers, arch.hidden_dim, arch.heads, 4 * arch.hidden_dim, norm)
        for mode in ("f16x3", "f16f8"):
            sc = E.PoetScorer(conf, st, 256, precision=mode)
            sc.set_context(ctx)
            k, v = sc.record(0)
            out[f"poet.norm{int(norm)}.{mode}.tok"] = sc.loglik(variants, tok_logp=True)[1]
            out[f"poet.norm{int(norm)}.{mode}.record0"] = np.concatenate([k.cpu().numpy(), v.cpu().numpy()], axis=1)
            sc.close()
    return out


def passes():
    """Runs with a max_rows small enough to split them into several passes, and ESM-1v wt-marginals of a 1 500-residue protein over
    overlapping 1024-token windows."""
    from proteingym_b200 import checkpoint, synth
    from proteingym_b200 import poet_engine as E
    from proteingym_b200.esm_engine import EsmScorer
    from proteingym_b200.progen3_engine import Progen3Scorer
    out = Runs()
    arch = synth.Progen3Arch(2, 256, 4, 2, 512)
    conf = checkpoint.progen3_config(arch.config())
    st = checkpoint.normalise_progen3_state(conf, synth.make_progen3_state(arch, 41))
    rng = np.random.default_rng(42)
    rows = [[1] + list(rng.integers(6, 34, n - 1)) for n in (5, 70, 130, 130, 300, 301, 301)]  # one batch of T = 301: three passes
    for mode in ("f16x3", "f16f8"):
        sc = Progen3Scorer(conf, st, precision=mode, max_rows=700)
        out[f"progen3.{mode}.passes"] = sc.token_sums(rows)
        sc.close()

    def row(n):
        return np.concatenate([[E.START], rng.integers(0, 20, size=n - 2), [E.STOP]]).astype(np.int64)
    ctx = [row(n) for n in (40, 130, 7, 90)]
    variants = [row(n) for n in (20, 65, 128, 129, 3, 100, 129)]  # T = 129: two rows per pass, four passes
    arch = synth.PoetArch(2, 256, 4, norm=True)
    st = synth.make_poet_state(arch, seed=43)
    conf = checkpoint.PoetConfig(arch.layers, arch.hidden_dim, arch.heads, 4 * arch.hidden_dim, True)
    for mode in ("f16x3", "f16f8"):
        sc = E.PoetScorer(conf, st, 256, precision=mode, max_rows=300)
        sc.set_context(ctx)
        out[f"poet.{mode}.passes.sum"] = sc.loglik(variants)
        out[f"poet.{mode}.passes.tok"] = sc.loglik(variants, tok_logp=True)[1]
        sc.close()
    arch = synth.EsmArch("esm1v", 2, 256, 4, 1024)
    sc = EsmScorer(checkpoint.config_from_synth(arch), checkpoint.normalise_synth_state(arch, synth.make_esm_state(arch, seed=44)),
                   precision="f16x3")
    out["esm1v.f16x3.wt_overlapping"] = sc.wt_marginal_table_overlapping(synth.random_protein(1500, 45)).cpu().numpy()
    sc.close()
    return out


def main():
    if sys.argv[1] == "--compare":
        a, b = np.load(sys.argv[2]), np.load(sys.argv[3])
        bad = [k for k in a.files if k not in b.files or not np.array_equal(a[k], b[k], equal_nan=True)] + [k for k in b.files if k not in a.files]
        for k in a.files:
            print(f"{k:40s} {a[k].shape} {'DIFFERENT' if k in bad else 'equal'}")
        sys.exit(1 if bad else 0)
    arrays = collect()
    assert all(np.isfinite(v).any() for v in arrays.values())
    np.savez(sys.argv[1], **arrays)
    print(f"wrote {len(arrays)} arrays to {sys.argv[1]}")


if __name__ == "__main__":
    main()
