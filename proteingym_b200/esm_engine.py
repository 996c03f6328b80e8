"""Host-side driver of the H100 ESM scorer: owns a libpgscore handle and exposes the two operations the reference's
masked-marginal path consists of (compute_fitness.py:486-514):

  * ``masked_marginal_table(seq)``   -> the ``token_probs`` [L+2, 33] table (one masked copy per token, batched), and
  * ``score_mutants(table, mutants)`` -> ``label_row`` over the whole DMS frame.

PyTorch is used for device memory and streams only; all arithmetic happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .alphabet import ALPHABET
from .checkpoint import EsmConfig, esmc_rotary_tables, rotary_tables
from .mutants import parse_esmc_mutants, parse_mutants
from .windows import esmc_window_rows, optimal_window_starts

PRECISIONS = {"f16": _lib.PG_PREC_F16, "f16x3": _lib.PG_PREC_F16X3, "f16f8": _lib.PG_PREC_F16F8, "f16d": _lib.PG_PREC_F16D}
ARCHS = {"esm1b": _lib.PG_ARCH_ESM1B, "esm2": _lib.PG_ARCH_ESM2, "esmc": _lib.PG_ARCH_ESMC}


def choose_precision(config: EsmConfig, mutants=None, strategy: str = "masked-marginals", seq_len: int = None) -> str:
    """``--precision auto``: the cheapest operand scheme whose MEASURED error meets the 1e-3 abs per-mutant bar for this job.

    f16f8 (2 tensor-pipe units) carries ~16-bit operands: per masked site its score error is 1.2e-4 mean / 4.5e-4 max at ESM-1v 650M
    (BLAT golden, 4997 mutants) and 6.1e-4 max at ESM2 3B; errors of independently masked sites add, so 5-site mutants reach 1.0e-3 at
    3B (tests/test_gpu_parity.py::test_golden_true_size_esm2_3b_multi_mutants). f16x3 (3 units, ~22-bit operands) stays at 8e-5 / 3.3e-4
    in the same tests. f16d (delta operands, 1 unit: shared base rows at x3 precision + one fp16 pass on the per-copy difference; built
    for the ESM-1b / ESM-1v masked-marginal pass over ONE shared window) measures 6.8e-5 mean / 3.9e-4 max on the same BLAT golden
    (286 residues). Its error scales with the size of the perturbation one mask causes, i.e. ~1/L: on a 96-residue protein it is
    7.6e-4 / 8.8e-4 / 1.5e-3 for 1 / 2 / 3 sites (f16f8: 3.4e-4 / 5.6e-4 / 6.0e-4; test_multi_site_error_growth_650m_vs_oracle), so
    short proteins stay on f16f8. ESM2 8M / 35M / 150M stay within 6.1e-4 in f16f8 (tests/test_gpu_esm2_small.py). ESM C (H100 80GB
    HBM3, goldens of the unmodified evoscale script at true size, tests/test_gpu_esmc.py) in f16f8: max score error 1.2e-4 (300M, 1- and
    2-site mutants), 1.4e-4 (600M), 9.9e-5 (300M, windowed L = 1150); f16x3 3.3e-5 / 4.9e-5 / 4.6e-5 — so ESM C follows the same rule
    (f16d is refused for it).
    Rule: for models up to 1280 wide when no mutant has more than two sites — f16d if the architecture and the strategy allow it and
    192 <= ``seq_len`` (residues; + 2 tokens must fit the 1024-token window), else f16f8; f16x3 otherwise."""
    if config.embed_dim > 1280:
        return "f16x3"
    if strategy == "pseudo-ppl":  # sums L rows per sequence
        return "f16x3"
    if mutants is not None:
        k = 0
        for m in mutants:
            c = m.count(":") + 1
            if c > k:
                k = c
                if k > 2:
                    return "f16x3"
    if config.arch == "esm1b" and strategy == "masked-marginals" and seq_len is not None and 192 <= seq_len <= config.max_positions - 2:
        return "f16d"
    return "f16f8"


class EsmScorer:
    def __init__(self, config: EsmConfig, state: dict, precision: str = "f16f8", device: int = 0, max_rows: int = 0):
        if not torch.cuda.is_available():
            raise _lib.PgError("no CUDA device: the H100 scorer has no CPU fallback")
        self.lib = _lib.load()
        self.config = config
        self.device = torch.device("cuda", device)
        self.precision = precision
        desc = _lib.PgModelDesc(
            arch=ARCHS[config.arch], layers=config.layers,
            embed_dim=config.embed_dim, heads=config.heads, ffn_dim=config.ffn_dim, vocab=config.vocab,
            max_positions=config.max_positions, token_dropout=int(config.token_dropout),
            emb_ln_before=int(config.emb_layer_norm_before), precision=PRECISIONS[precision], device=device,
            max_rows=max_rows)
        self.handle = C.c_void_p()
        _lib.check(self.lib.pg_create(C.byref(desc), C.byref(self.handle)))
        try:
            self._upload(state)
        except Exception:
            self.close()
            raise

    def _upload(self, state: dict):
        cfg = self.config
        tensors = {k: v for k, v in state.items() if "rot_emb.inv_freq" not in k}
        if cfg.arch == "esm2":
            inv = state["layers.0.self_attn.rot_emb.inv_freq"]
            cos, sin = rotary_tables(inv, 16384)  # rotary has no length limit in the reference; 16384 tokens covers every ProteinGym target (max 3423)
            tensors["rotary.cos"], tensors["rotary.sin"] = cos, sin
        elif cfg.arch == "esmc":
            tensors["rotary.cos"], tensors["rotary.sin"] = esmc_rotary_tables(1024)  # every ESM C window is <= 1024 tokens
        # fp32 staging copy on the device (ESM-1v 2.6 GB, ESM2-3B 11 GB); the library repacks and we free it
        gpu = [(n, t.to(self.device, torch.float32).contiguous()) for n, t in tensors.items()]
        arr = (_lib.PgTensor * len(gpu))()
        for i, (n, t) in enumerate(gpu):
            arr[i].name = n.encode()
            arr[i].data = t.data_ptr()
            arr[i].shape[0] = t.shape[0]
            arr[i].shape[1] = t.shape[1] if t.dim() == 2 else 1
        torch.cuda.synchronize(self.device)
        _lib.check(self.lib.pg_load_weights(self.handle, arr, len(gpu)), self.handle)
        del gpu
        torch.cuda.empty_cache()

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle:
            self.lib.pg_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------------------
    def masked_marginal_rows(self, tokens: torch.Tensor, positions, model_window: int = 1024) -> torch.Tensor:
        """log_softmax rows [P, 33] for the given masked token indices (device int32 ``tokens`` of the full sequence).
        Windows follow the reference's ``--scoring-window optimal`` rule (compute_fitness.py:492-495)."""
        n_tokens = int(tokens.numel())
        pos_np = np.asarray(positions, dtype=np.int32)
        starts_np, T = optimal_window_starts(pos_np, n_tokens, model_window)
        P = len(pos_np)
        out = torch.empty((P, self.config.vocab), dtype=torch.float32, device=self.device)
        if P == 0:
            return out
        stage = torch.from_numpy(np.stack([pos_np, starts_np])).to(self.device, non_blocking=True)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        windowed = n_tokens > model_window
        _lib.check(self.lib.pg_masked_marginals(self.handle, tokens.data_ptr(), n_tokens, stage[0].data_ptr(),
                                                stage[1].data_ptr() if windowed else None, None, P, T,
                                                out.data_ptr(), stream), self.handle)
        self._keepalive = stage
        return out

    def masked_marginal_table(self, sequence: str, positions=None, model_window: int = 1024) -> torch.Tensor:
        """The reference's ``token_probs[0]``: [L+2, 33] on the device. ``positions`` (token indices, BOS = 0) restricts
        the work to the rows ``label_row`` will actually read; other rows are NaN. Default: every residue position
        (the reference also runs the BOS/EOS copies, whose rows no mutant can address)."""
        tok_np = ALPHABET.tokenize_sequence(sequence)
        tokens = torch.from_numpy(tok_np).to(self.device)
        if positions is None:
            positions = np.arange(1, len(sequence) + 1, dtype=np.int32)
        positions = np.asarray(positions, dtype=np.int32)
        if self.config.arch == "esmc" and len(sequence) > model_window - 2:  # compute_fitness.py:346-409: re-tokenised windows
            if len(positions) and (positions.min() < 1 or positions.max() > len(sequence)):
                raise IndexError("ESM C windows hold residue positions 1..L only")
            rows = self.esmc_rows(sequence, positions - 1, model_window)
        else:
            rows = self.masked_marginal_rows(tokens, positions, model_window)
        table = torch.full((len(tok_np), self.config.vocab), float("nan"), dtype=torch.float32, device=self.device)
        table[torch.from_numpy(positions.astype(np.int64)).to(self.device)] = rows
        return table

    def esmc_rows(self, sequence: str, seq_positions, window_size: int = 1024) -> torch.Tensor:
        """ESM C: log_softmax rows [P, 64] with residue ``seq_positions[p]`` (0-based) masked in its window (one token row per distinct
        ``<cls> slice <eos>`` window, windows.esmc_window_rows)."""
        res = ALPHABET.tokenize_sequence(sequence)[1:-1]
        tok, pos, starts, T = esmc_window_rows(res, seq_positions, ALPHABET.cls_idx, ALPHABET.eos_idx, window_size)
        P = len(pos)
        out = torch.empty((P, self.config.vocab), dtype=torch.float32, device=self.device)
        if P == 0:
            return out
        stage = torch.from_numpy(np.concatenate([tok, pos, starts])).to(self.device)
        n = len(tok)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.pg_masked_marginals(self.handle, stage.data_ptr(), n, stage[n:].data_ptr(), stage[n + P:].data_ptr(), None,
                                                P, T, out.data_ptr(), stream), self.handle)
        self._keepalive = stage
        return out

    def wt_marginal_table(self, sequence: str) -> torch.Tensor:
        """One unmasked forward, log_softmax of every token (compute_fitness.py:475)."""
        tok_np = ALPHABET.tokenize_sequence(sequence)
        tokens = torch.from_numpy(tok_np).to(self.device)
        out = torch.empty((len(tok_np), self.config.vocab), dtype=torch.float32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.pg_forward_logprobs(self.handle, tokens.data_ptr(), len(tok_np), 0, len(tok_np), -1,
                                                out.data_ptr(), stream), self.handle)
        return out

    def _forward_window(self, tokens: torch.Tensor, start: int, T: int, mask_pos: int = -1) -> torch.Tensor:
        out = torch.empty((T, self.config.vocab), dtype=torch.float32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.pg_forward_logprobs(self.handle, tokens.data_ptr(), int(tokens.numel()), start, T, mask_pos,
                                                out.data_ptr(), stream), self.handle)
        return out

    def wt_marginal_table_overlapping(self, sequence: str) -> torch.Tensor:
        """``--scoring-window overlapping`` for wt-marginals on sequences longer than 1024 tokens
        (compute_fitness.py:435-473): sigmoid-tapered 1024-token windows sliding in from both ends by 511, plus a central
        window when the final overlap is under 511; weighted average of the windows' log-softmax rows. The forwards run
        in the CUDA library; the [T,33] weighted accumulation is host-orchestrated torch glue, as in the reference."""
        import math
        tok_np = ALPHABET.tokenize_sequence(sequence)
        tokens = torch.from_numpy(tok_np).to(self.device)
        n = len(tok_np)
        probs = torch.zeros((n, self.config.vocab), dtype=torch.float32, device=self.device)
        wsum = torch.zeros((n,), dtype=torch.float32, device=self.device)
        w = torch.ones(1024)
        for i in range(1, 257):
            w[i] = 1 / (1 + math.exp(-(i - 128) / 16))
        for i in range(1022 - 256, 1023):
            w[i] = 1 / (1 + math.exp((i - 1022 + 128) / 16))
        w = w.to(self.device)

        def add(start):
            lp = self._forward_window(tokens, start, 1024)
            probs[start:start + 1024] += lp * w.view(-1, 1)
            wsum[start:start + 1024] += w

        sl, el = 0, 1023
        sr, er = (n - 1) - 1024 + 1, n - 1
        while True:
            add(sl)
            add(sr)
            if el > sr:
                break
            sl += 511; el += 511; sr -= 511; er -= 511
        if el - sr + 1 < 511:
            add(int(n / 2) - 512)
        return probs / wsum.view(-1, 1)

    def pseudo_ppl(self, sequence: str) -> float:
        """``compute_pppl`` (compute_fitness.py:258-279), including its indexing: for i in 1..len-2 mask TOKEN i and read
        the log-probability of ``sequence[i]`` there. No windowing (the reference has none for this strategy)."""
        tok_np = ALPHABET.tokenize_sequence(sequence)
        tokens = torch.from_numpy(tok_np).to(self.device)
        idx = list(range(1, len(sequence) - 1))
        if not idx:
            return 0
        rows = self.masked_marginal_rows(tokens, idx, model_window=max(len(tok_np), 1024)).cpu()
        return sum(rows[r, ALPHABET.get_idx(sequence[i])].item() for r, i in enumerate(idx))

    # ------------------------------------------------------------------------------------------------------------
    def prepare_assay(self, sequence: str, mutants, offset_idx: int = 1, model_window: int = 1024, pinned: bool = True):
        """Host half of one assay: tokenise, parse mutants, find which token rows ``label_row`` will read and their
        windows. Returns pinned host arrays + sizes; nothing touches the device. ESM C follows its own script's rules instead
        (evoscale compute_fitness.py:69-136, 346-409): no offset, invalid mutants skipped (NaN), re-tokenised windows."""
        if self.config.arch == "esmc":
            return self._prepare_assay_esmc(sequence, mutants, model_window, pinned)
        tok = ALPHABET.tokenize_sequence(sequence)
        site_row, site_wt, site_mt, offs = parse_mutants(mutants, sequence, offset_idx)
        if len(site_row) and (site_row.min() < 1 or site_row.max() > len(sequence)):
            raise IndexError("mutation position outside the sequence")
        positions = np.unique(site_row).astype(np.int32)            # exact pruning: only rows some mutant reads
        starts, T = optimal_window_starts(positions, len(tok), model_window)
        row_of = np.full(len(tok), -1, dtype=np.int32)
        row_of[positions] = np.arange(len(positions), dtype=np.int32)
        site_trow = row_of[site_row]                                  # index into the compact [P, vocab] table
        packed = np.concatenate([tok, positions, starts, site_trow, site_wt, site_mt, offs]).astype(np.int32)
        host = torch.from_numpy(packed)
        if pinned:
            host = host.pin_memory()
        sizes = dict(n_tokens=len(tok), P=len(positions), T=T, S=len(site_row), M=len(offs) - 1,
                     windowed=len(tok) > model_window)
        return host, sizes

    def _prepare_assay_esmc(self, sequence: str, mutants, window_size: int, pinned: bool):
        site_pos, site_wt, site_mt, offs, valid = parse_esmc_mutants(mutants, sequence)
        seq_pos = np.unique(site_pos).astype(np.int32)
        res = ALPHABET.tokenize_sequence(sequence)[1:-1]
        tok, positions, starts, T = esmc_window_rows(res, seq_pos, ALPHABET.cls_idx, ALPHABET.eos_idx, window_size)
        row_of = np.full(len(sequence) + 1, -1, dtype=np.int32)
        row_of[seq_pos] = np.arange(len(seq_pos), dtype=np.int32)
        packed = np.concatenate([tok, positions, starts, row_of[site_pos], site_wt, site_mt, offs]).astype(np.int32)
        host = torch.from_numpy(packed)
        if pinned:
            host = host.pin_memory()
        sizes = dict(n_tokens=len(tok), P=len(seq_pos), T=T, S=len(site_pos), M=len(offs) - 1, windowed=True,
                     invalid=np.flatnonzero(~valid))
        return host, sizes

    def run_assay(self, host: torch.Tensor, sizes: dict, dev: torch.Tensor | None = None, shard=None) -> torch.Tensor:
        """Device half: (optional H2D of the packed int32 block) -> masked-marginal rows -> mutant scores [M] (device).
        Pass ``dev`` to reuse an already-resident copy of ``host`` (bench's HBM-resident leg). ``shard = (rank, world)`` with an
        initialised torch.distributed group: this rank computes only its contiguous chunk of the P masked positions and the
        [P, vocab] table is completed by one all-gather (position partitioning of a single assay, SURVEY.md §8e)."""
        if dev is None:
            dev = host.to(self.device, non_blocking=True)
        n, P, T, S, M = sizes["n_tokens"], sizes["P"], sizes["T"], sizes["S"], sizes["M"]
        o = [0, n, n + P, n + 2 * P, n + 2 * P + S, n + 2 * P + 2 * S, n + 2 * P + 3 * S]
        tok, pos, st, trow, wt, mt, offs = (dev[o[i]:(o[i + 1] if i + 1 < len(o) else None)] for i in range(7))
        stream = torch.cuda.current_stream(self.device).cuda_stream
        lo, hi, rows = 0, P, max(P, 1)
        if shard is not None:
            from . import sharding
            lo, hi, chunk = sharding.position_chunk(P, shard[1], shard[0])
            rows = max(shard[1] * chunk, 1)
        table = torch.empty((rows, self.config.vocab), dtype=torch.float32, device=self.device)
        scores = torch.empty((M,), dtype=torch.float32, device=self.device)
        if hi > lo:
            _lib.check(self.lib.pg_masked_marginals(self.handle, tok.data_ptr(), n, pos[lo:].data_ptr(),
                                                    st[lo:].data_ptr() if sizes["windowed"] else None, None, hi - lo, T,
                                                    table[lo:].data_ptr(), stream), self.handle)
        if shard is not None:
            sharding.all_gather_rows(table, chunk)
        if M:
            _lib.check(self.lib.pg_score_mutants(table.data_ptr(), P, self.config.vocab, trow.data_ptr(), wt.data_ptr(),
                                                 mt.data_ptr(), offs.data_ptr(), M, scores.data_ptr(), stream))
        invalid = sizes.get("invalid")
        if invalid is not None and len(invalid):  # mutants the reference skips get NaN (evoscale compute_fitness.py:592)
            scores[torch.from_numpy(invalid).to(self.device)] = float("nan")
        self._keepalive3 = (dev, table)
        return scores

    def score_assay(self, sequence: str, mutants, offset_idx: int = 1, model_window: int = 1024, shard=None) -> np.ndarray:
        """Public one-call API: WT sequence + mutant strings in, per-mutant scores (host float32) out — what
        compute_fitness.py:486-514 does for one checkpoint. ``shard``: see run_assay (every rank returns all the scores)."""
        host, sizes = self.prepare_assay(sequence, mutants, offset_idx, model_window)
        scores = self.run_assay(host, sizes, shard=shard)
        out = torch.empty(scores.shape, dtype=torch.float32).pin_memory()
        out.copy_(scores, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return out.numpy()

    def score_mutants(self, table: torch.Tensor, mutants, sequence: str, offset_idx: int = 1) -> torch.Tensor:
        """``df.apply(label_row)`` for all rows at once (compute_fitness.py:505-514) -> float32 [M] on the device."""
        site_row, site_wt, site_mt, offs = parse_mutants(mutants, sequence, offset_idx)
        M = len(offs) - 1
        out = torch.empty((M,), dtype=torch.float32, device=self.device)
        if M == 0:
            return out
        if len(site_row) and (site_row.min() < 0 or site_row.max() >= table.shape[0]):
            raise IndexError("mutation position outside the sequence")
        dev = lambda a: torch.from_numpy(a).to(self.device, non_blocking=True)
        d_row, d_wt, d_mt, d_off = dev(site_row), dev(site_wt), dev(site_mt), dev(offs)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.pg_score_mutants(table.data_ptr(), table.shape[0], table.shape[1], d_row.data_ptr(),
                                             d_wt.data_ptr(), d_mt.data_ptr(), d_off.data_ptr(), M, out.data_ptr(),
                                             stream))
        self._keepalive2 = (d_row, d_wt, d_mt, d_off)
        return out
