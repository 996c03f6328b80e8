"""fair-esm checkpoint reader for the H100 scorer (host side, replaces the model-construction half of
``pretrained.load_model_and_alphabet``; reference: proteingym/baselines/esm/esm/pretrained.py:24-28,67-77,85-99,
162-181,184-218).

Returns a flat fp32 state (reference key names with the ``encoder.`` / ``encoder.sentence_encoder.`` prefixes removed)
plus the architecture description the C-ABI needs. Nothing here builds an nn.Module.
"""
from __future__ import annotations

import argparse
import os
import re
from dataclasses import dataclass
from pathlib import Path

import torch

MASK_IDX = 32


@dataclass
class EsmConfig:
    arch: str            # "esm1b" (ESM-1b / ESM-1v, learned positions) | "esm2" (rotary) | "msa" (MSA Transformer) | "esmc" (ESM C)
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    token_dropout: bool
    emb_layer_norm_before: bool
    max_positions: int = 1024
    vocab: int = 33


def _strip_v1(name: str) -> str:
    # pretrained.py:90-93: drop everything up to and including "encoder." / "sentence_encoder."
    if "sentence_encoder." in name:
        name = "".join(name.split("sentence_encoder.")[1:])
    if "encoder." in name:
        name = "".join(name.split("encoder.")[1:])
    return name


def checkpoint_column_name(model_location: str) -> str:
    """Name of the score column a checkpoint produces: the reference's ``model_location.split("/")[-1].split(".")[0]``
    (compute_fitness.py:350), i.e. everything before the FIRST dot of the file name (``esm1v.v2.pt`` -> ``esm1v``)."""
    return os.path.basename(str(model_location)).split(".")[0]


def load_esm_checkpoint(model_location: str):
    """-> (EsmConfig, state: dict[str, fp32 CPU tensor], score column name)."""
    path = Path(model_location)
    if not str(model_location).endswith(".pt"):
        raise ValueError("only local .pt checkpoints are supported (no network): " + str(model_location))
    with torch.serialization.safe_globals([argparse.Namespace]):
        data = torch.load(str(path), map_location="cpu", weights_only=True)
    name = path.stem
    if name.startswith("esm2"):  # pretrained.py:187
        cfg = data["cfg"]["model"]
        pat = re.compile("^" + "|".join(["encoder.sentence_encoder.", "encoder."]))
        raw = {pat.sub("", k): v for k, v in data["model"].items()}
        conf = EsmConfig("esm2", int(cfg.encoder_layers), int(cfg.encoder_embed_dim), int(cfg.encoder_attention_heads),
                         4 * int(cfg.encoder_embed_dim), bool(cfg.token_dropout), False)
    else:
        args = data["args"]
        if args.arch != "roberta_large":
            raise ValueError(f"unsupported fair-esm architecture {args.arch!r} (ESM-1b/ESM-1v/ESM2 only)")
        raw = {_strip_v1(k): v for k, v in data["model"].items()}
        get = lambda n, dflt=None: getattr(args, n, getattr(args, "encoder_" + n, dflt))
        # pretrained.py:97: zero the <mask> embedding in place ("for token drop"); aliasing with lm_head.weight is kept
        raw["embed_tokens.weight"][MASK_IDX].zero_()
        conf = EsmConfig("esm1b", int(get("layers")), int(get("embed_dim")), int(get("attention_heads")),
                         int(get("ffn_embed_dim")), bool(getattr(args, "token_dropout", False)),
                         any(k.startswith("emb_layer_norm_before") for k in raw), int(get("max_positions", 1024)))
    # The tied output matrix: load_state_dict copies "lm_head.weight" into the shared parameter after
    # "embed_tokens.weight" (lm_head is registered last, esm1.py:97-101 / esm2.py:70-74), so it wins.
    tied = raw["lm_head.weight"] if "lm_head.weight" in raw else raw["embed_tokens.weight"]
    state = {k: v.detach().to(torch.float32).contiguous() for k, v in raw.items()
             if not k.startswith("contact_head") and k != "lm_head.weight"}
    state["embed_tokens.weight"] = tied.detach().to(torch.float32).contiguous()
    return conf, state, checkpoint_column_name(model_location)


def _msa_model_key(name: str) -> str:
    """File key -> model key of an msa_transformer checkpoint (pretrained.py:107-115): the loader swaps "row" and "column" in every
    name (the first release stored the two attention blocks under each other's names), then strips the encoder prefixes."""
    if "row" in name:
        name = name.replace("row", "column")
    else:
        name = name.replace("column", "row")
    return _strip_v1(name)


def load_msa_checkpoint(model_location: str):
    """-> (EsmConfig with arch "msa", state: dict[str, fp32 CPU tensor], score column name) for a fair-esm ``msa_transformer`` file.
    ``msa_position_embedding`` is returned as [1024, embed_dim] (the first release's [1, 1024, 1, 1] table broadcasts over the width,
    msa_transformer.py:166-168); absent when the checkpoint was trained without it."""
    path = Path(model_location)
    if not str(model_location).endswith(".pt"):
        raise ValueError("only local .pt checkpoints are supported (no network): " + str(model_location))
    with torch.serialization.safe_globals([argparse.Namespace]):
        data = torch.load(str(path), map_location="cpu", weights_only=True)
    args = data["args"]
    if args.arch != "msa_transformer":
        raise ValueError(f"not an msa_transformer checkpoint: {args.arch!r}")
    raw = {_msa_model_key(k): v for k, v in data["model"].items()}
    get = lambda n, dflt=None: getattr(args, n, getattr(args, "encoder_" + n, dflt))
    conf = EsmConfig("msa", int(get("layers")), int(get("embed_dim")), int(get("attention_heads")), int(get("ffn_embed_dim")),
                     False, True, int(get("max_positions", 1024)))
    tied = raw["lm_head.weight"] if "lm_head.weight" in raw else raw["embed_tokens.weight"]
    state = {k: v.detach().to(torch.float32).contiguous() for k, v in raw.items()
             if not k.startswith("contact_head") and k != "lm_head.weight"}
    state["embed_tokens.weight"] = tied.detach().to(torch.float32).contiguous()
    if get("embed_positions_msa", False) and "msa_position_embedding" in state:
        state["msa_position_embedding"] = normalise_row_positions(state["msa_position_embedding"], conf.embed_dim)
    else:
        state.pop("msa_position_embedding", None)
    return conf, state, checkpoint_column_name(model_location)


def normalise_row_positions(t: torch.Tensor, d: int) -> torch.Tensor:
    t = t.to(torch.float32).reshape(1024, -1)
    return t.expand(1024, d).contiguous()


def config_from_msa_synth(arch) -> EsmConfig:
    return EsmConfig("msa", arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, False, True, arch.max_positions, arch.vocab)


def normalise_msa_synth_state(arch, st: dict) -> dict:
    """Apply to an in-memory ``synth.make_msa_state`` dict what ``load_msa_checkpoint`` does to a file."""
    st = {k: v.to(torch.float32).contiguous() for k, v in st.items() if k != "lm_head.weight"}
    if "msa_position_embedding" in st:
        st["msa_position_embedding"] = normalise_row_positions(st["msa_position_embedding"], arch.embed_dim)
    return st


def config_from_synth(arch) -> EsmConfig:
    """EsmConfig for a ``synth.EsmArch`` (tests / bench build states in memory instead of writing 2.6 GB files)."""
    return EsmConfig("esm2" if arch.kind == "esm2" else "esm1b", arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim,
                     arch.token_dropout, arch.emb_layer_norm_before, arch.max_positions, arch.vocab)


def normalise_synth_state(arch, st: dict) -> dict:
    """Apply to an in-memory ``synth.make_esm_state`` dict what ``load_esm_checkpoint`` does to a file."""
    st = {k: v.clone() for k, v in st.items()}
    if arch.kind != "esm2":
        st["embed_tokens.weight"][MASK_IDX].zero_()
    st.pop("lm_head.weight", None)  # tied alias of embed_tokens.weight in synth states
    return {k: v.to(torch.float32).contiguous() for k, v in st.items()}


def rotary_tables(inv_freq: torch.Tensor, T: int):
    """cos/sin [T, 32] exactly as the reference builds them (esm/rotary_embedding.py:46-61): fp32 outer product of
    arange(T) with the checkpoint's ``inv_freq`` buffer, then cos / sin. Both halves of the 64-wide table are equal."""
    t = torch.arange(T).type_as(inv_freq)
    freqs = torch.einsum("i,j->ij", t, inv_freq.float())
    return freqs.cos().contiguous(), freqs.sin().contiguous()


# ESM C releases (evoscale esm/pretrained.py:65-98; f = swiglu_correction_fn(8/3, d), esm/layers/blocks.py:15-17):
# name -> (layers, d_model, SwiGLU hidden width f, weight file under the snapshot root)
ESMC_RELEASES = {"esmc_300M": (30, 960, 2560, "data/weights/esmc_300m_2024_12_v0.pth"),
                 "esmc_600M": (36, 1152, 3072, "data/weights/esmc_600m_2024_12_v0.pth")}
ESMC_HF_REPOS = {"esmc_300M": "EvolutionaryScale/esmc-300m-2024-12", "esmc_600M": "EvolutionaryScale/esmc-600m-2024-12"}


def esmc_config_from_state(state: dict) -> EsmConfig:
    """Dims of an ESM C state dict from its shapes: d from ``embed.weight`` [64, d], layers from the block keys, f from
    ``ffn.1.weight`` [2f, d]; checks every key the scorer reads and its shape."""
    d = int(state["embed.weight"].shape[1])
    if state["embed.weight"].shape[0] != 64 or d % 64:
        raise ValueError("ESM C: embed.weight must be [64, d] with d a multiple of 64 (head_dim 64)")
    layers = 1 + max(int(k.split(".")[2]) for k in state if k.startswith("transformer.blocks."))
    f = int(state["transformer.blocks.0.ffn.1.weight"].shape[0]) // 2
    want = {"embed.weight": (64, d), "transformer.norm.weight": (d,), "sequence_head.0.weight": (d, d), "sequence_head.0.bias": (d,),
            "sequence_head.2.weight": (d,), "sequence_head.2.bias": (d,), "sequence_head.3.weight": (64, d), "sequence_head.3.bias": (64,)}
    for i in range(layers):
        p = f"transformer.blocks.{i}."
        want.update({p + "attn.layernorm_qkv.0.weight": (d,), p + "attn.layernorm_qkv.0.bias": (d,),
                     p + "attn.layernorm_qkv.1.weight": (3 * d, d), p + "attn.q_ln.weight": (d,), p + "attn.k_ln.weight": (d,),
                     p + "attn.out_proj.weight": (d, d), p + "ffn.0.weight": (d,), p + "ffn.0.bias": (d,),
                     p + "ffn.1.weight": (2 * f, d), p + "ffn.3.weight": (d, f)})
    for k, shape in want.items():
        if k not in state:
            raise ValueError(f"ESM C state dict: missing {k}")
        if tuple(state[k].shape) != shape:
            raise ValueError(f"ESM C state dict: {k} has shape {tuple(state[k].shape)}, expected {shape}")
    return EsmConfig("esmc", layers, d, d // 64, f, False, False, 1024, 64)


def resolve_esmc_weights(model_type: str, model_path: str | None = None) -> str:
    """``--model_path`` as the .pth file itself or a snapshot directory holding ``data/weights/esmc_*_2024_12_v0.pth``; without it, the
    local Hugging Face cache (HF_HUB_CACHE / HF_HOME / ~/.cache/huggingface). Never downloads."""
    rel = ESMC_RELEASES[model_type][3]
    if model_path:
        p = Path(model_path)
        if p.is_file():
            return str(p)
        if (p / rel).is_file():
            return str(p / rel)
        raise FileNotFoundError(f"{model_path}: neither an ESM C .pth file nor a directory holding {rel}")
    hub = os.environ.get("HF_HUB_CACHE") or os.path.join(os.environ.get("HF_HOME") or os.path.expanduser("~/.cache/huggingface"), "hub")
    snaps = Path(hub) / ("models--" + ESMC_HF_REPOS[model_type].replace("/", "--")) / "snapshots"
    found = sorted(snaps.glob("*/" + rel)) if snaps.is_dir() else []
    if not found:
        raise FileNotFoundError(f"{model_type} weights not found in the local Hugging Face cache ({snaps}); pass --model_path "
                                f"(a {os.path.basename(rel)} file or a snapshot directory). Weights are never downloaded.")
    return str(found[-1])


def load_esmc_checkpoint(model_type: str, model_path: str | None = None):
    """-> (EsmConfig with arch "esmc", state: dict[str, fp32 CPU tensor] with the reference key names, score column name
    ``{model_type}_score``). Reads the .pth state dict (weights_only) and checks its dims against the release table."""
    if model_type not in ESMC_RELEASES:
        raise ValueError(f"unknown ESM C release {model_type!r} (esmc_300M, esmc_600M)")
    path = resolve_esmc_weights(model_type, model_path)
    raw = torch.load(path, map_location="cpu", weights_only=True)
    state = {k: v.detach().to(torch.float32).contiguous() for k, v in raw.items()}
    conf = esmc_config_from_state(state)
    layers, d, f, _ = ESMC_RELEASES[model_type]
    if (conf.layers, conf.embed_dim, conf.ffn_dim) != (layers, d, f):
        raise ValueError(f"{path}: dims (layers {conf.layers}, d {conf.embed_dim}, f {conf.ffn_dim}) are not {model_type}'s "
                         f"({layers}, {d}, {f})")
    return conf, state, f"{model_type}_score"


def esmc_rotary_tables(T: int = 1024):
    """cos/sin [T, 32] of ESM C's rotary (esm/layers/rotary.py:136-165): inv_freq = 1 / 10000^(arange(0, 64, 2) / 64) in fp32,
    torch.outer with arange(T) in fp32, then cos / sin."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64))
    freqs = torch.outer(torch.arange(T, dtype=torch.float32), inv_freq)
    return freqs.cos().contiguous(), freqs.sin().contiguous()


# ---- RITA (proteingym/baselines/rita: rita_configuration.py, rita_modeling.py) ----------------------------------------------------
def _read_hf_weights(folder: str) -> dict:
    """The state dict of a Hugging Face model directory: pytorch_model.bin, else every *.safetensors file."""
    pbin = os.path.join(folder, "pytorch_model.bin")
    if os.path.exists(pbin):
        return torch.load(pbin, map_location="cpu", weights_only=True)
    st_files = sorted(Path(folder).glob("*.safetensors"))
    if not st_files:
        raise FileNotFoundError(f"{folder}: neither pytorch_model.bin nor *.safetensors")
    from safetensors.torch import load_file
    raw = {}
    for f in st_files:
        raw.update(load_file(str(f)))
    return raw


@dataclass
class RitaConfig:
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    vocab: int
    tied: bool               # the output head is the embedding matrix


def load_rita_checkpoint(folder: str):
    """RITA model directory -> (RitaConfig, state, inv_freq). ``state`` has the key names of include/pgscore.h's PG_ARCH_RITA (the
    ``transformer.`` prefix stripped, no rotary buffers) as fp32 CPU tensors; ``inv_freq`` is the checkpoint's rotary buffer.

    config.json: ``d_model``, ``num_layers``, ``num_heads``, ``ff_ratio`` (the FFN width is d_model * ff_ratio, rita_configuration.py:
    25-26), ``vocab_size`` and ``tie_word_embeddings``, with RITAConfig's defaults for absent keys. Weights: pytorch_model.bin or
    *.safetensors.

    Head tying follows the rule of PretrainedConfig in the transformers release the reference pins (4.32.1): ``tie_word_embeddings``
    defaults to true, and ``from_pretrained`` then ties ``lm_head.weight`` to the embedding. That release could not be inspected here
    (DESIGN.md §2 records this assumption and what would change it); an ``lm_head.weight`` that tying discards and that differs from
    the embedding is reported with a warning. With ``"tie_word_embeddings": false`` the checkpoint's ``lm_head.weight`` is the head."""
    import json
    import warnings
    cfg = json.load(open(os.path.join(folder, "config.json")))
    raw = _read_hf_weights(folder)
    d, layers, heads = int(cfg.get("d_model", 768)), int(cfg.get("num_layers", 12)), int(cfg.get("num_heads", 12))
    ffn, vocab = d * int(cfg.get("ff_ratio", 4)), int(cfg.get("vocab_size", 26))
    tied = bool(cfg.get("tie_word_embeddings", True))
    state, inv = {}, []
    for k, v in raw.items():
        name = k[len("transformer."):] if k.startswith("transformer.") else k
        if name.endswith("rotary_embedding.inv_freq"):
            inv.append((name, v.float()))
            continue
        state[name] = v.detach().float().contiguous()
    if len(inv) != layers:
        raise ValueError(f"{folder}: {len(inv)} rotary_embedding.inv_freq buffers for {layers} layers")
    inv_freq = inv[0][1]
    for name, t in inv[1:]:
        if t.shape != inv_freq.shape or not torch.equal(t, inv_freq):
            raise ValueError(f"{folder}: {name} differs from {inv[0][0]}: the layers disagree on the rotary frequencies")
    if tied:
        head = state.pop("lm_head.weight", None)
        if head is not None and not torch.equal(head, state.get("embedding.weight", head)):
            warnings.warn(f"{folder}: lm_head.weight differs from the embedding and is discarded: config.json does not set "
                          "tie_word_embeddings to false, so the head is tied to the embedding")
    elif "lm_head.weight" not in state:
        raise ValueError(f"{folder}: tie_word_embeddings is false but the checkpoint has no lm_head.weight")
    want = {"embedding.weight": (vocab, d), "final_norm.weight": (d,), "final_norm.bias": (d,)}
    if not tied:
        want["lm_head.weight"] = (vocab, d)
    for i in range(layers):
        p = f"layers.{i}."
        for nm in ("query", "key", "value", "proj"):
            want[p + f"self_attention.{nm}.weight"] = (d, d)
            want[p + f"self_attention.{nm}.bias"] = (d,)
        want.update({p + "attn_norm.weight": (d,), p + "attn_norm.bias": (d,), p + "mlp_norm.weight": (d,), p + "mlp_norm.bias": (d,),
                     p + "mlp.0.weight": (ffn, d), p + "mlp.0.bias": (ffn,), p + "mlp.2.weight": (d, ffn), p + "mlp.2.bias": (d,)})
    for k, shape in want.items():
        if k not in state:
            raise ValueError(f"RITA state dict: missing {k}")
        if tuple(state[k].shape) != shape:
            raise ValueError(f"RITA state dict: {k} has shape {tuple(state[k].shape)}, expected {shape}")
    if d % heads or inv_freq.numel() != (d // heads) // 2:
        raise ValueError(f"RITA: d_model {d} / num_heads {heads} does not match inv_freq of {inv_freq.numel()} frequencies")
    return RitaConfig(layers, d, heads, ffn, vocab, tied), state, inv_freq


@dataclass
class Progen2Config:
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    vocab: int
    rotary_dim: int          # rotary dims per head, from the front of each head (modeling_progen.py:178-186)
    n_positions: int         # the scorer's chunk length (compute_fitness.py:163)

    @property
    def head_dim(self) -> int:
        return self.embed_dim // self.heads


def load_progen2_checkpoint(folder: str):
    """ProGen2 model directory -> (Progen2Config, state). ``state`` has the key names of include/pgscore.h's PG_ARCH_PROGEN2 (the
    ``transformer.`` prefix stripped, the causal-mask buffers ``attn.bias`` / ``attn.masked_bias`` dropped) as fp32 CPU tensors, any
    stored dtype upcast.

    config.json: ``n_embd``, ``n_layer``, ``n_head``, ``rotary_dim``, ``n_inner``, ``n_positions``, ``vocab_size``, ``layer_norm_epsilon``
    and ``activation_function``, with ProGenConfig's defaults for absent keys (configuration_progen.py:26-46). Weights:
    pytorch_model.bin or *.safetensors. What the kernels do not implement is refused: LayerNorm eps other than 1e-5, an activation other
    than gelu_new, head_dim > 128 (progen2-xlarge), a vocabulary without the scored columns 5..29."""
    import json
    cfg = json.load(open(os.path.join(folder, "config.json")))
    raw = _read_hf_weights(folder)
    d, layers, heads = int(cfg.get("n_embd", 4096)), int(cfg.get("n_layer", 28)), int(cfg.get("n_head", 16))
    vocab, npos = int(cfg.get("vocab_size", 50400)), int(cfg.get("n_positions", 2048))
    ffn = int(cfg["n_inner"]) if cfg.get("n_inner") is not None else 4 * d
    eps = float(cfg.get("layer_norm_epsilon", 1e-5))
    act = cfg.get("activation_function", "gelu_new")
    if d % heads:
        raise ValueError(f"ProGen2: n_embd {d} is not a multiple of n_head {heads}")
    hd = d // heads
    rot = cfg.get("rotary_dim", 64)
    if rot is None:  # the attention would rotate the whole head (:187-190), but ProGenModel.__init__ fails first (:325)
        raise ValueError("ProGen2: rotary_dim null: the reference's ProGenModel cannot be built with it (modeling_progen.py:325)")
    rot = int(rot)
    if eps != 1e-5:
        raise NotImplementedError(f"ProGen2: layer_norm_epsilon {eps}: the LayerNorm kernels use eps 1e-5")
    if act != "gelu_new":
        raise NotImplementedError(f"ProGen2: activation_function {act!r}: the MLP epilogue implements gelu_new (tanh GELU)")
    if hd > 128:
        raise NotImplementedError(f"ProGen2: head_dim {hd} (n_embd {d} / n_head {heads}, progen2-xlarge) has no attention tile (at most 128)")
    if rot % 2 or not 0 < rot <= hd:
        raise ValueError(f"ProGen2: rotary_dim {rot} must be even and within head_dim {hd}")
    if vocab < 30:
        raise ValueError(f"ProGen2: vocab_size {vocab} lacks the scored token ids 5..29")
    state = {}
    for k, v in raw.items():
        name = k[len("transformer."):] if k.startswith("transformer.") else k
        if name.endswith("attn.bias") or name.endswith("attn.masked_bias"):
            continue
        state[name] = v.detach().float().contiguous()
    want = {"wte.weight": (vocab, d), "ln_f.weight": (d,), "ln_f.bias": (d,), "lm_head.weight": (vocab, d), "lm_head.bias": (vocab,)}
    for i in range(layers):
        p = f"h.{i}."
        want.update({p + "ln_1.weight": (d,), p + "ln_1.bias": (d,), p + "attn.qkv_proj.weight": (3 * d, d),
                     p + "attn.out_proj.weight": (d, d), p + "mlp.fc_in.weight": (ffn, d), p + "mlp.fc_in.bias": (ffn,),
                     p + "mlp.fc_out.weight": (d, ffn), p + "mlp.fc_out.bias": (d,)})
    for k, shape in want.items():
        if k not in state:
            raise ValueError(f"ProGen2 state dict: missing {k}")
        if tuple(state[k].shape) != shape:
            raise ValueError(f"ProGen2 state dict: {k} has shape {tuple(state[k].shape)}, expected {shape}")
    extra = sorted(set(state) - set(want))
    if extra:
        raise ValueError(f"ProGen2 state dict: unexpected keys {extra[:5]}")
    return Progen2Config(layers, d, heads, ffn, vocab, rot, npos), state


def progen2_rotary_tables(rotary_dim: int, slot: int, T: int):
    """cos/sin [T, slot/2] for the library's rotary epilogue: columns i < rotary_dim/2 hold sin / cos(t * inv_freq[i]) computed as
    fixed_pos_embedding does (modeling_progen.py:38-44: inv_freq = 1 / 10000^(arange(0, dim, 2) / dim) and the outer product in fp32),
    the others cos = 1, sin = 0 (dims that pass through unrotated)."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, rotary_dim, 2) / rotary_dim))
    sinusoid = torch.einsum("i , j -> i j", torch.arange(T), inv_freq).float()
    cos, sin = torch.ones((T, slot // 2)), torch.zeros((T, slot // 2))
    cos[:, :rotary_dim // 2], sin[:, :rotary_dim // 2] = torch.cos(sinusoid), torch.sin(sinusoid)
    return cos.contiguous(), sin.contiguous()


@dataclass
class Protgpt2Config:
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    vocab: int
    n_positions: int         # rows of the learned position table


def load_protgpt2_checkpoint(folder: str):
    """ProtGPT2 (GPT-2) model directory -> (Protgpt2Config, state). ``state`` has the key names of include/pgscore.h's PG_ARCH_PROTGPT2
    (the ``transformer.`` prefix stripped; the tied ``lm_head.weight`` and the causal-mask buffers ``attn.bias`` / ``attn.masked_bias``
    dropped) as fp32 CPU tensors; Conv1D weights stay [in, out].

    config.json: ``n_embd``, ``n_layer``, ``n_head``, ``n_inner``, ``n_positions``, ``vocab_size``, ``layer_norm_epsilon``,
    ``activation_function``, ``scale_attn_weights``, ``scale_attn_by_inverse_layer_idx`` and ``tie_word_embeddings``, with GPT2Config's
    defaults for absent keys. Weights: pytorch_model.bin or *.safetensors. What the kernels do not implement is refused: an activation
    other than gelu_new, LayerNorm eps other than 1e-5, attention scaled by the layer index or not scaled, head_dim other than 64, an
    untied head."""
    import json
    cfg = json.load(open(os.path.join(folder, "config.json")))
    d, layers, heads = int(cfg.get("n_embd", 768)), int(cfg.get("n_layer", 12)), int(cfg.get("n_head", 12))
    vocab, npos = int(cfg.get("vocab_size", 50257)), int(cfg.get("n_positions", 1024))
    ffn = int(cfg["n_inner"]) if cfg.get("n_inner") is not None else 4 * d
    act = cfg.get("activation_function", "gelu_new")
    eps = float(cfg.get("layer_norm_epsilon", 1e-5))
    if act != "gelu_new":
        raise NotImplementedError(f"ProtGPT2: activation_function {act!r}: the MLP epilogue implements gelu_new (tanh GELU)")
    if eps != 1e-5:
        raise NotImplementedError(f"ProtGPT2: layer_norm_epsilon {eps}: the LayerNorm kernels use eps 1e-5")
    if cfg.get("scale_attn_by_inverse_layer_idx", False):
        raise NotImplementedError("ProtGPT2: scale_attn_by_inverse_layer_idx: the attention scale is folded as 1/sqrt(head_dim) only")
    if not cfg.get("scale_attn_weights", True):
        raise NotImplementedError("ProtGPT2: scale_attn_weights false: the attention scale 1/sqrt(head_dim) is folded into q")
    if not cfg.get("tie_word_embeddings", True):
        raise NotImplementedError("ProtGPT2: tie_word_embeddings false: the fused head is the tied wte")
    if d % heads or d // heads != 64:
        raise NotImplementedError(f"ProtGPT2: head_dim {d / heads:g} (n_embd {d} / n_head {heads}): the kernels take 64-wide heads")
    if d % 64 or ffn % 64:
        raise NotImplementedError(f"ProtGPT2: n_embd {d} and n_inner {ffn} must be multiples of 64 (GEMM K tiles)")
    raw = _read_hf_weights(folder)
    state = {}
    for k, v in raw.items():
        name = k[len("transformer."):] if k.startswith("transformer.") else k
        if name.endswith(".attn.bias") or name.endswith(".attn.masked_bias") or name == "lm_head.weight":
            continue
        state[name] = v.detach().float().contiguous()
    want = {"wte.weight": (vocab, d), "wpe.weight": (npos, d), "ln_f.weight": (d,), "ln_f.bias": (d,)}
    for i in range(layers):
        p = f"h.{i}."
        want.update({p + "ln_1.weight": (d,), p + "ln_1.bias": (d,), p + "ln_2.weight": (d,), p + "ln_2.bias": (d,),
                     p + "attn.c_attn.weight": (d, 3 * d), p + "attn.c_attn.bias": (3 * d,), p + "attn.c_proj.weight": (d, d),
                     p + "attn.c_proj.bias": (d,), p + "mlp.c_fc.weight": (d, ffn), p + "mlp.c_fc.bias": (ffn,),
                     p + "mlp.c_proj.weight": (ffn, d), p + "mlp.c_proj.bias": (d,)})
    for k, shape in want.items():
        if k not in state:
            raise ValueError(f"ProtGPT2 state dict: missing {k}")
        if tuple(state[k].shape) != shape:
            raise ValueError(f"ProtGPT2 state dict: {k} has shape {tuple(state[k].shape)}, expected {shape}")
    extra = sorted(set(state) - set(want))
    if extra:
        raise ValueError(f"ProtGPT2 state dict: unexpected keys {extra[:5]}")
    return Protgpt2Config(layers, d, heads, ffn, vocab, npos), state
