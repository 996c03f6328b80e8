"""The checks every scoring entry point makes before it launches anything, on one small seeded handle per family (ESM, MSA Transformer,
decoder, PoET): a handle of another family and a handle without weights get PG_ERR_STATE, a ProGen3 handle refuses a retrieval prior
with PG_ERR_ARG and wild-type prefix reuse with PG_ERR_UNSUPPORTED."""
import ctypes as C

import pytest
import torch

from proteingym_b200 import _lib, checkpoint, msa_engine, synth

pytestmark = pytest.mark.gpu

PG_ERR_ARG, PG_ERR_STATE, PG_ERR_UNSUPPORTED = 1, 3, 4


def esm():
    from proteingym_b200.esm_engine import EsmScorer
    a = synth.EsmArch("esm1v", 1, 128, 2, 256)
    return EsmScorer(checkpoint.config_from_synth(a), checkpoint.normalise_synth_state(a, synth.make_esm_state(a, 1)), max_rows=4096)


def msa():
    a = synth.MsaArch(1, 128, 2, 256)
    return msa_engine.MsaScorer(checkpoint.config_from_msa_synth(a), checkpoint.normalise_msa_synth_state(a, synth.make_msa_state(a, 2)),
                                max_rows=4096)


def decoder():
    from proteingym_b200.progen3_engine import Progen3Scorer
    a = synth.Progen3Arch(1, 128, 2, 1, 256)
    conf = checkpoint.progen3_config(a.config())
    return Progen3Scorer(conf, checkpoint.normalise_progen3_state(conf, synth.make_progen3_state(a, 3)), max_rows=4096)


def poet():
    from proteingym_b200.poet_engine import PoetScorer
    a = synth.PoetArch(1, 128, 2, norm=True)
    return PoetScorer(checkpoint.PoetConfig(a.layers, a.hidden_dim, a.heads, 4 * a.hidden_dim, True), synth.make_poet_state(a, 4), 256,
                      max_rows=4096)


FAMILIES = {"esm": esm, "msa": msa, "decoder": decoder, "poet": poet}


class Bufs:
    """Device buffers larger than any call below reads or writes, zero-filled."""

    def __init__(self):
        self.keep = [torch.zeros(1 << 16, dtype=torch.int32, device="cuda"), torch.zeros(1 << 16, device="cuda"),
                     torch.full((4,), 8, dtype=torch.int32, device="cuda")]
        self.i, self.f, self.lens = (t.data_ptr() for t in self.keep)


# entry point -> (the family it runs, a call with valid sizes on handle h)
CALLS = {
    "pg_masked_marginals": ("esm", lambda lib, h, b: lib.pg_masked_marginals(h, b.i, 8, b.i, None, None, 2, 8, b.f, None)),
    "pg_forward_logprobs": ("esm", lambda lib, h, b: lib.pg_forward_logprobs(h, b.i, 8, 0, 8, -1, b.f, None)),
    "pg_msa_masked_marginals": ("msa", lambda lib, h, b: lib.pg_msa_masked_marginals(h, b.i, 2, 8, b.i, None, 1, 8, b.f, None)),
    "pg_ar_loglik": ("decoder", lambda lib, h, b: lib.pg_ar_loglik(h, b.i, b.lens, 1, 8, None, None, 0.0, b.f, None)),
    "pg_ar_loglik_fused": ("decoder", lambda lib, h, b: lib.pg_ar_loglik_fused(h, b.i, b.lens, 1, 8, None, b.f, None)),
    "pg_ar_prefix_begin": ("decoder", lambda lib, h, b: lib.pg_ar_prefix_begin(h, b.i, 8, None, b.f, None)),
    "pg_ar_loglik_prefix": ("decoder", lambda lib, h, b: lib.pg_ar_loglik_prefix(h, b.i, b.lens, 1, 8, 128, None, b.f, None)),
    "pg_progen3_routing": ("decoder", lambda lib, h, b: lib.pg_progen3_routing(h, 0, b.i, b.f, C.byref(C.c_int32()), None)),
    "pg_poet_context": ("poet", lambda lib, h, b: lib.pg_poet_context(h, b.i, (C.c_int32 * 1)(8), 1, None)),
    "pg_poet_loglik": ("poet", lambda lib, h, b: lib.pg_poet_loglik(h, b.i, b.lens, 1, 8, b.f, None, None)),
    "pg_poet_record": ("poet", lambda lib, h, b: lib.pg_poet_record(h, 0, b.f, 1 << 12, None)),
}


@pytest.fixture(scope="module")
def handles():
    """family -> (its loaded scorer, the PgModelDesc it was created from)."""
    seen, made = {}, {}
    init = _lib.Model.__init__

    def spy(self, desc, tensors, device=0):
        seen["desc"] = desc
        init(self, desc, tensors, device)
    _lib.Model.__init__ = spy
    try:
        for fam, make in FAMILIES.items():
            made[fam] = (make(), seen["desc"])
    finally:
        _lib.Model.__init__ = init
    yield made
    for sc, _ in made.values():
        sc.close()


def refused(lib, call, handle, code):
    """call(handle) returns `code` and launches nothing; -> its error message."""
    b = Bufs()
    torch.cuda.synchronize()
    n0 = lib.pg_launch_count()
    assert call(lib, handle, b) == code
    torch.cuda.synchronize()
    assert lib.pg_launch_count() == n0
    return lib.pg_last_error(handle).decode()


@pytest.mark.parametrize("entry,fam", [(e, f) for e in CALLS for f in FAMILIES if f != CALLS[e][0]])
def test_wrong_family_is_refused(handles, entry, fam):
    msg = refused(_lib.load(), CALLS[entry][1], handles[fam][0].handle, PG_ERR_STATE)
    assert "handle is" in msg, msg


@pytest.mark.parametrize("entry", [e for e in CALLS if e not in ("pg_poet_record", "pg_progen3_routing")])  # readers of a record
def test_handle_without_weights_is_refused(handles, entry):
    lib = _lib.load()
    h = C.c_void_p()
    _lib.check(lib.pg_create(C.byref(handles[CALLS[entry][0]][1]), C.byref(h)))
    try:
        assert "weights not loaded" in refused(lib, CALLS[entry][1], h, PG_ERR_STATE)
    finally:
        lib.pg_destroy(h)


def test_progen3_refuses_a_retrieval_prior(handles):
    lib, h = _lib.load(), handles["decoder"][0].handle
    fused = lambda lib, h, b: lib.pg_ar_loglik_fused(  # noqa: E731
        h, b.i, b.lens, 1, 8, C.byref(_lib.PgArFusion(log_prior=b.f, prior_row=b.i, alpha=0.5)), b.f, None)
    plain = lambda lib, h, b: lib.pg_ar_loglik(h, b.i, b.lens, 1, 8, b.f, b.i, 0.5, b.f, None)  # noqa: E731
    for call in (fused, plain):
        assert "ProGen3 has no retrieval fusion" in refused(lib, call, h, PG_ERR_ARG)


def test_progen3_refuses_prefix_reuse(handles):
    lib, h = _lib.load(), handles["decoder"][0].handle
    assert "ProGen3" in refused(lib, CALLS["pg_ar_prefix_begin"][1], h, PG_ERR_UNSUPPORTED)
