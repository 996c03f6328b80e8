"""Host-side driver of the H100 MSA Transformer scorer: alignment sampling as the reference does it, tokenisation, and the batched
masked-marginal table (reference: proteingym/baselines/esm/compute_fitness.py:26-98 sampling, :360-425 scoring loop;
esm/data.py:300-336 MSABatchConverter). PyTorch is used for device memory and streams only; the arithmetic is in libpgscore.so.
"""
from __future__ import annotations

import itertools
import random

import numpy as np
import torch

from . import _lib
from .alphabet import ALPHABET
from .checkpoint import EsmConfig
from .mutants import parse_mutants
from .windows import optimal_window_starts


def read_fasta_records(path):
    """(description, sequence) per record in file order — what ``SeqIO.parse(path, "fasta")`` yields to the reference (:31-37)."""
    name, parts = None, []
    with open(path) as fh:
        for line in fh:
            line = line.rstrip("\n")
            if line.startswith(">"):
                if name is not None:
                    yield name, "".join(parts)
                name, parts = line[1:], []
            elif name is not None:
                parts.append(line.strip())
    if name is not None:
        yield name, "".join(parts)


def process_msa(filename: str, weight_filename, filter_msa: bool = False, device: int = 0):
    """``process_msa`` (:76-98): the EVE-style alignment object with sequence weights (read from ``weight_filename`` or computed on
    the GPU and saved there). ``--filter-msa`` shells out to hhfilter in the reference; that external binary is not reproduced."""
    if filter_msa:
        raise NotImplementedError("--filter-msa runs the external hhfilter binary in the reference (compute_fitness.py:78-89); "
                                  "filter the alignment beforehand and pass the filtered file")
    from .msa_processing import MSAProcessing
    # defaults of proteingym/utils/msa_utils.py:25-38 (focus-column threshold 1.0: every column of the target stays a focus column)
    msa = MSAProcessing(MSA_location=filename, use_weights=True, weights_location=weight_filename, threshold_focus_cols_frac_gaps=1.0,
                        device=device, on_missing_weights="compute")
    print("Name of focus_seq: " + str(msa.focus_seq_name))
    return msa


def sample_msa(filename: str, nseq: int, sampling_strategy: str, random_seed: int, weight_filename=None, processed_msa=None, device: int = 0):
    """``sample_msa`` (:26-73): the rows of the alignment the model sees, target first. Python's ``random`` is used on purpose: the
    reference seeds it and calls ``random.sample`` / ``random.choices``, so the same seed gives the same rows."""
    print("Sampling sequences from MSA with strategy: " + str(sampling_strategy))
    random.seed(random_seed)
    if sampling_strategy == "first_x_rows":
        msa = list(itertools.islice(read_fasta_records(filename), nseq))
    elif sampling_strategy == "random":
        msa = list(read_fasta_records(filename))
        nseq = min(len(msa), nseq)
        msa = random.sample(msa, nseq)
    elif sampling_strategy == "sequence-reweighting":
        MSA = processed_msa if processed_msa is not None else process_msa(filename, weight_filename, device=device)
        msa = [(MSA.focus_seq_name, MSA.raw_seq_name_to_sequence[MSA.focus_seq_name])]
        non_wt_weights = np.array([w for k, w in MSA.seq_name_to_weight.items() if k != MSA.focus_seq_name])
        non_wt_sequences = [(k, s) for k, s in MSA.seq_name_to_sequence.items() if k != MSA.focus_seq_name]
        non_wt_weights = non_wt_weights / non_wt_weights.sum()
        if len(non_wt_sequences) > 0:
            msa.extend(random.choices(non_wt_sequences, weights=non_wt_weights, k=nseq - 1))
        print("Check sum weights MSA: " + str(non_wt_weights.sum()))
    else:
        raise UnboundLocalError("unknown --msa-sampling-strategy " + str(sampling_strategy))  # the reference leaves `msa` unbound (:70)
    msa = [(desc, "".join(seq) if isinstance(seq, list) else seq) for desc, seq in msa]
    return [(desc, seq.upper()) for desc, seq in msa]


def tokenize_alignment(rows) -> np.ndarray:
    """MSABatchConverter for one alignment (data.py:300-336; prepend_bos, no eos): [(name, aligned string)] -> int32 [R, L + 1]."""
    L = len(rows[0][1])
    if any(len(s) != L for _, s in rows):
        raise RuntimeError("Received unaligned sequences for input to MSA, all sequence lengths must be equal.")
    out = np.empty((len(rows), L + 1), dtype=np.int32)
    out[:, 0] = ALPHABET.cls_idx
    for r, (_, s) in enumerate(rows):
        out[r, 1:] = ALPHABET.encode(s)
    return out


def default_max_rows(config: EsmConfig, R: int, Cw: int, np_planes: int = 2, budget_bytes: float = 40e9, want: int = 4) -> int:
    """Workspace rows for ``want`` masked alignments per pass, fewer when that would not fit ``budget_bytes`` of HBM (residual stream,
    operand buffers, q/k/v, MLP hidden and the tied-attention regroupings: ~(10 + 8 np) d + 2 np f bytes per token row)."""
    d, f = config.embed_dim, config.ffn_dim
    per_row = 4 * d + 2 * np_planes * d + 6 * np_planes * d + 2 * np_planes * f + 8 * np_planes * d
    per_msa = R * Cw
    n = max(1, min(want, int(budget_bytes // (per_row * per_msa))))
    return n * per_msa


class MsaScorer(_lib.Model):
    def __init__(self, config: EsmConfig, state: dict, precision: str = "f16x3", device: int = 0, max_rows: int = 0):
        if config.arch != "msa":
            raise ValueError("MsaScorer needs an MSA Transformer configuration")
        self.config = config
        self.precision = precision
        self.max_rows = int(max_rows)
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_MSA, layers=config.layers, embed_dim=config.embed_dim, heads=config.heads,
                                ffn_dim=config.ffn_dim, vocab=config.vocab, max_positions=config.max_positions, token_dropout=0,
                                emb_ln_before=1, precision=_lib.PRECISIONS[precision], device=device, max_rows=max_rows)
        super().__init__(desc, state, device)

    # ------------------------------------------------------------------------------------------------------------
    def masked_marginal_rows(self, tokens: np.ndarray, positions, shard=None) -> torch.Tensor:
        """The reference loop body (:383-399) for the given columns of row 0: tokens int32 [R, C] (BOS column included) ->
        float32 [len(positions), vocab] on the device, row p = log_softmax(logits[0, 0, positions[p]]) with (0, positions[p]) masked.
        Alignments wider than 1024 columns use the reference's per-position window (``get_optimal_window`` with L + 2, :389).
        ``shard = (rank, world)`` with an initialised torch.distributed group: the masked positions are independent forwards, so this
        rank runs a contiguous chunk of them and one all-gather completes the table on every rank (SURVEY.md §8e)."""
        if shard is not None and shard[1] > 1:
            from . import sharding
            positions = np.asarray(positions, dtype=np.int32)
            lo, hi, chunk = sharding.position_chunk(len(positions), shard[1], shard[0])
            full = torch.zeros((shard[1] * chunk, self.config.vocab), dtype=torch.float32, device=self.device)
            if hi > lo:
                full[lo:hi] = self.masked_marginal_rows(tokens, positions[lo:hi])
            return sharding.all_gather_rows(full, chunk)[:len(positions)]
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        R, Cf = tokens.shape
        if (tokens == ALPHABET.padding_idx).any():
            raise ValueError("padding tokens in the alignment: rows of one alignment have equal length on this path")
        positions = np.asarray(positions, dtype=np.int32)
        out = torch.empty((len(positions), self.config.vocab), dtype=torch.float32, device=self.device)
        if len(positions) == 0:
            return out
        if positions.min() < 0 or positions.max() >= Cf:
            raise IndexError("masked column outside the alignment")
        dev_tok = torch.from_numpy(tokens).to(self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if Cf > 1024:
            starts, _ = optimal_window_starts(positions, Cf + 1, 1024)      # the reference passes len(sequence) + 2 = C + 1
            widths = np.minimum(starts + 1024, Cf) - starts                   # the slice [start:end] is clipped at C
        else:
            starts, widths = np.zeros(len(positions), dtype=np.int32), np.full(len(positions), Cf, dtype=np.int64)
        for w in np.unique(widths):
            sel = np.flatnonzero(widths == w)
            pos = torch.from_numpy(positions[sel]).to(self.device)
            st = torch.from_numpy(starts[sel].astype(np.int32)).to(self.device)
            part = torch.empty((len(sel), self.config.vocab), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_msa_masked_marginals(self.handle, dev_tok.data_ptr(), R, Cf, pos.data_ptr(),
                                                        st.data_ptr() if Cf > 1024 else None, len(sel), int(w), part.data_ptr(), stream),
                       self.handle)
            out[torch.from_numpy(sel).to(self.device)] = part
        self._keep = (dev_tok,)
        return out

    def score_assay(self, rows, sequence: str, mutants, offset_idx: int = 1, shard=None) -> np.ndarray:
        """One (checkpoint, seed) column (:377-405): ``rows`` = the sampled alignment [(name, aligned string)], ``sequence`` = the part
        of the target the alignment covers, ``offset_idx`` = MSA_start. Only the columns some mutant reads are forwarded (exact)."""
        tokens = tokenize_alignment(rows)
        site_row, site_wt, site_mt, offs = parse_mutants(mutants, sequence, offset_idx)
        # label_row indexes token_probs[0, 1 + idx] with Python / torch semantics (:248-249): a position before MSA_start gives a negative
        # index that wraps to the end of the alignment (and its wild-type check reads sequence[idx] the same way); reproduced as is
        site_row = np.where(site_row < 0, site_row + tokens.shape[1], site_row).astype(np.int32)
        if len(site_row) and (site_row.min() < 0 or site_row.max() >= tokens.shape[1]):
            raise IndexError("mutation position outside the alignment")
        positions = np.unique(site_row).astype(np.int32)
        table = self.masked_marginal_rows(tokens, positions, shard=shard)
        row_of = np.full(tokens.shape[1], -1, dtype=np.int32)
        row_of[positions] = np.arange(len(positions), dtype=np.int32)
        M = len(offs) - 1
        scores = torch.empty((M,), dtype=torch.float32, device=self.device)
        if M:
            dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(self.device)
            d_row, d_wt, d_mt, d_off = dev(row_of[site_row]), dev(site_wt), dev(site_mt), dev(offs)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(self.lib.pg_score_mutants(table.data_ptr(), len(positions), self.config.vocab, d_row.data_ptr(), d_wt.data_ptr(),
                                                 d_mt.data_ptr(), d_off.data_ptr(), M, scores.data_ptr(), stream))
        return scores.cpu().numpy()
