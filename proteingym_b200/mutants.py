"""Mutant-string parsing to flat int32 site arrays (host half of ``label_row``,
reference: proteingym/baselines/esm/compute_fitness.py:240-250)."""
from __future__ import annotations

import re

import numpy as np

from .alphabet import ALPHABET


def parse_mutants(mutants, sequence: str, offset_idx: int = 1):
    """-> (site_row, site_wt, site_mt, row_offsets) int32 arrays in CSR form.

    ``site_row`` is the token index ``1 + idx`` (BOS shifts by one, compute_fitness.py:248-249). Raises
    ``AssertionError("The listed wildtype does not match the provided sequence")`` exactly where the reference does
    (:244), and ``ValueError`` / ``IndexError`` for malformed entries like the reference's ``int()`` / indexing would."""
    rows, wts, mts, offs = [], [], [], [0]
    get_idx = ALPHABET.get_idx
    for row in mutants:
        for mutation in str(row).split(":"):
            wt, idx, mt = mutation[0], int(mutation[1:-1]) - offset_idx, mutation[-1]
            assert sequence[idx] == wt, "The listed wildtype does not match the provided sequence"
            rows.append(1 + idx)
            wts.append(get_idx(wt))
            mts.append(get_idx(mt))
        offs.append(len(rows))
    as32 = lambda a: np.asarray(a, dtype=np.int32)
    return as32(rows), as32(wts), as32(mts), as32(offs)


_ESMC_SITE = re.compile(r"([A-Z])(\d+)([A-Z])")
_ESMC_AA = "ACDEFGHIKLMNPQRSTVWY"


def parse_esmc_mutants(mutants, sequence: str):
    """ESM C's mutant handling (evoscale compute_fitness.py:69-136, 310-320, 427-472) -> (site_pos, site_wt, site_mt, row_offsets,
    valid) with ``site_pos`` the 0-based residue index (no offset: positions are 1-based) and ``valid`` [M] bool.

    Every ':'-separated site must ``re.match`` ``([A-Z])(\\d+)([A-Z])``, lie inside the sequence and name the sequence's residue as
    wild type; a mutant failing any of these is skipped (no sites, ``valid`` False: NaN in the reference's CSV). The wt / mt letters
    of a kept site index a table of the 20 amino acids; any other letter raises ``KeyError`` as the reference's lookup does."""
    pos, wts, mts, offs, valid = [], [], [], [0], []
    get_idx = ALPHABET.get_idx
    for row in mutants:
        sites = []
        for sub in str(row).split(":"):
            m = _ESMC_SITE.match(sub)
            if not m:
                sites = None
                break
            wt, p, mt = m.group(1), int(m.group(2)) - 1, m.group(3)
            if p < 0 or p >= len(sequence) or sequence[p] != wt:
                sites = None
                break
            sites.append((p, wt, mt))
        if sites is not None:
            for p, wt, mt in sites:
                if wt not in _ESMC_AA or mt not in _ESMC_AA:
                    raise KeyError(wt if wt not in _ESMC_AA else mt)
                pos.append(p)
                wts.append(get_idx(wt))
                mts.append(get_idx(mt))
        valid.append(sites is not None)
        offs.append(len(pos))
    as32 = lambda a: np.asarray(a, dtype=np.int32)
    return as32(pos), as32(wts), as32(mts), as32(offs), np.asarray(valid, dtype=bool)
