"""pg_load_weights on one seeded one-layer model per architecture: every tensor role it reads is checked (a dropped tensor and a
mis-shaped one are named in the error), a handle loads once, and the ESM masked-marginal calls refuse handles of other
architectures before launching anything."""
import ctypes as C
import os

import pytest
import torch

from proteingym_b200 import _lib, checkpoint, msa_engine, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PG_ERR_ARG, PG_ERR_STATE = 1, 3


def _strip(st):
    return {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()}


def esm1b():
    from proteingym_b200.esm_engine import EsmScorer
    a = synth.EsmArch("esm1v", 1, 128, 2, 256, emb_layer_norm_before=True)
    return EsmScorer(checkpoint.config_from_synth(a), checkpoint.normalise_synth_state(a, synth.make_esm_state(a, 1)), max_rows=4096)


def esm2():
    from proteingym_b200.esm_engine import EsmScorer
    a = synth.EsmArch("esm2", 1, 160, 4, 256)
    return EsmScorer(checkpoint.config_from_synth(a), checkpoint.normalise_synth_state(a, synth.make_esm_state(a, 2)), max_rows=4096)


def esmc():
    from proteingym_b200.esm_engine import EsmScorer
    st = synth.make_esmc_state(synth.EsmcArch(1, 128, 256), seed=3)
    return EsmScorer(checkpoint.esmc_config_from_state(st), st, max_rows=4096)


def msa():
    a = synth.MsaArch(1, 128, 2, 256)
    return msa_engine.MsaScorer(checkpoint.config_from_msa_synth(a), checkpoint.normalise_msa_synth_state(a, synth.make_msa_state(a, 4)),
                                max_rows=4096)


def tranception():
    from proteingym_b200.tranception_engine import TranceptionScorer
    a = synth.TranceptionArch(1, 256, 4, 512)
    cfg = {"n_embd": 256, "n_head": 4, "n_layer": 1, "n_ctx": 1024, "n_inner": 512, "vocab_size": 25, "layer_norm_epsilon": 1e-5,
           "activation_function": "squared_relu"}
    st = {k[len("transformer."):]: v for k, v in synth.make_tranception_state(a, 5).items() if k.startswith("transformer.")}
    return TranceptionScorer(cfg, st, max_rows=4096)


def rita():
    from proteingym_b200.rita_engine import RitaScorer, RitaTokenizer
    a = synth.RitaArch(1, 128, 2)
    st = synth.make_rita_state(a, 6, untied=True)
    ws = {k: v for k, v in _strip(st).items() if "inv_freq" not in k}
    return RitaScorer(checkpoint.RitaConfig(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, False), ws,
                      st["transformer.layers.0.self_attention.rotary_embedding.inv_freq"],
                      RitaTokenizer(os.path.join(GOLDEN, "rita_tokenizer_plain")), max_rows=4096)


def progen2():
    from proteingym_b200.progen2_engine import Progen2Scorer
    a = synth.Progen2Arch(1, 640, 8, 32)  # 80-wide heads in 128-wide slots
    return Progen2Scorer(checkpoint.Progen2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.rotary_dim, a.n_positions),
                         _strip(synth.make_progen2_state(a, 7, buffers=False)), max_rows=4096)


def protgpt2():
    from proteingym_b200.protgpt2_engine import Protgpt2Scorer, Protgpt2Tokenizer
    a = synth.Protgpt2Arch(1, 128, 2)
    ws = {k: v for k, v in _strip(synth.make_protgpt2_state(a, 8)).items() if k != "lm_head.weight"}
    return Protgpt2Scorer(checkpoint.Protgpt2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.n_positions), ws,
                          Protgpt2Tokenizer(os.path.join(GOLDEN, "protgpt2_tokenizer")), max_rows=4096)


def poet():
    from proteingym_b200.poet_engine import PoetScorer
    a = synth.PoetArch(1, 128, 2, norm=True)
    return PoetScorer(checkpoint.PoetConfig(a.layers, a.hidden_dim, a.heads, 4 * a.hidden_dim, True), synth.make_poet_state(a, 9), 256,
                      max_rows=4096)


# per architecture: its scorer, and one tensor of each role pg_load_weights reads (attention weight, LayerNorm, embedding, rotary table
# or the architecture's own extra)
ARCHS = {
    "esm1b": (esm1b, ["layers.0.self_attn.q_proj.weight", "layers.0.final_layer_norm.bias", "embed_tokens.weight",
                      "emb_layer_norm_before.weight"]),
    "esm2": (esm2, ["layers.0.self_attn.v_proj.weight", "emb_layer_norm_after.weight", "embed_tokens.weight", "rotary.cos"]),
    "esmc": (esmc, ["transformer.blocks.0.attn.layernorm_qkv.1.weight", "transformer.blocks.0.attn.k_ln.weight", "embed.weight",
                    "rotary.sin"]),
    "msa": (msa, ["layers.0.column_self_attention.layer.k_proj.weight", "layers.0.row_self_attention.layer_norm.weight",
                  "embed_tokens.weight", "embed_positions.weight"]),
    "tranception": (tranception, ["h.0.attn.c_attn.weight", "h.0.ln_2.bias", "wte.weight", "h.0.attn.conv_taps"]),
    "rita": (rita, ["layers.0.self_attention.key.weight", "layers.0.attn_norm.weight", "embedding.weight", "rotary.cos"]),
    "progen2": (progen2, ["h.0.attn.qkv_proj.weight", "ln_f.weight", "wte.weight", "rotary.sin"]),
    "protgpt2": (protgpt2, ["h.0.attn.c_proj.weight", "h.0.ln_1.weight", "wte.weight", "wpe.weight"]),
    "poet": (poet, ["decoder.layers.0.multihead_attn.q_proj.weight", "decoder.layers.0.norm2.bias", "token_embed.weight", "rotary.cos"]),
}
LN_ROLE = 1  # index of the LayerNorm tensor in each list above


def _inputs(name, monkeypatch):
    """The PgModelDesc and the tensors the architecture's scorer hands the library (the scorer itself is closed again)."""
    seen = {}
    init = _lib.Model.__init__

    def spy(self, desc, tensors, device=0):
        seen["desc"], seen["tensors"] = desc, dict(tensors)
        init(self, desc, tensors, device)
    with monkeypatch.context() as m:
        m.setattr(_lib.Model, "__init__", spy)
        ARCHS[name][0]().close()
    return seen["desc"], seen["tensors"]


def _stage(tensors):
    """The pg_tensor array of `tensors` (fp32, on the device) and the device tensors it points into."""
    gpu = [(n, t.to("cuda", torch.float32).contiguous()) for n, t in tensors.items()]
    arr = (_lib.PgTensor * len(gpu))()
    for i, (n, t) in enumerate(gpu):
        arr[i].name, arr[i].data = n.encode(), t.data_ptr()
        arr[i].shape[0], arr[i].shape[1] = t.shape[0], t.shape[1] if t.dim() == 2 else 1
    torch.cuda.synchronize()
    return arr, gpu


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ARCHS))
def test_missing_and_misshaped_tensors_are_named(name, monkeypatch):
    desc, tensors = _inputs(name, monkeypatch)
    for role in ARCHS[name][1]:
        assert role in tensors, role
        bad = {k: v for k, v in tensors.items() if k != role}
        with pytest.raises(_lib.PgError, match="missing or mis-shaped tensors") as e:
            _lib.Model(desc, bad)
        assert role in str(e.value), (role, str(e.value))
    role = ARCHS[name][1][LN_ROLE]
    bad = dict(tensors)
    bad[role] = tensors[role][:-1]
    with pytest.raises(_lib.PgError, match="missing or mis-shaped tensors") as e:
        _lib.Model(desc, bad)
    assert f"{role}(shape)" in str(e.value), str(e.value)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ARCHS))
def test_one_load_per_handle(name, monkeypatch):
    desc, tensors = _inputs(name, monkeypatch)
    lib = _lib.load()
    arr, keep = _stage(tensors)
    m = _lib.Model(desc, tensors)  # loaded
    try:
        assert lib.pg_load_weights(m.handle, arr, len(arr)) == PG_ERR_STATE
        assert b"one load per handle" in lib.pg_last_error(m.handle)
    finally:
        m.close()
    role = ARCHS[name][1][0]
    bad, keep_bad = _stage({k: v for k, v in tensors.items() if k != role})
    h = C.c_void_p()
    _lib.check(lib.pg_create(C.byref(desc), C.byref(h)))
    try:  # a failed load leaves the handle unusable too
        assert lib.pg_load_weights(h, bad, len(bad)) == PG_ERR_ARG
        assert lib.pg_load_weights(h, arr, len(arr)) == PG_ERR_STATE
    finally:
        lib.pg_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["poet", "rita", "msa"])
def test_masked_marginals_refuse_other_architectures(name):
    lib = _lib.load()
    sc = ARCHS[name][0]()
    try:
        T = 16
        tokens = torch.full((T,), 4, dtype=torch.int32, device="cuda")
        positions = torch.arange(1, 3, dtype=torch.int32, device="cuda")
        out = torch.zeros((T, 64), dtype=torch.float32, device="cuda")
        n0 = lib.pg_launch_count()
        assert lib.pg_masked_marginals(sc.handle, tokens.data_ptr(), T, positions.data_ptr(), None, None, 2, T, out.data_ptr(),
                                       sc.stream()) == PG_ERR_STATE
        assert lib.pg_forward_logprobs(sc.handle, tokens.data_ptr(), T, 0, T, -1, out.data_ptr(), sc.stream()) == PG_ERR_STATE
        assert b"handle is" in lib.pg_last_error(sc.handle)
        torch.cuda.synchronize()
        assert lib.pg_launch_count() == n0
        assert (out == 0).all()
    finally:
        sc.close()
