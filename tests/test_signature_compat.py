"""Drop-in proof: every name, keyword and positional order the reference uses must bind against this repo's mirrors.
The reference's API surface is stored in tests/golden/reference_signatures.json, read from its sources (never imported --
they need FlashInfer and the compiled pybind modules) by tests/golden/make_golden.py.

  * `models/attnserver.py` class LSHSparseAttnServer (reference :7-331): constructor parameters with defaults and the
    seven methods with their parameter names -> `magicpig_b200.attnserver.LSHSparseAttnServer`.
  * `models/llama.py` call sites (:91-93 constructor keywords, :208, 264, 282-284, 292, 315, 357 method calls):
    every call is replayed with `inspect.Signature.bind` on the mirror.
  * pybind `.def(...)` lists (`library/lsh/lsh.cc:316-326`, `library/sparse_attention/sparse_attention.cc:1243-1263`)
    and the C++ member declarations (`lsh.h:18-27`, `sparse_attention.h:19-35`) -> `magicpig_b200.ops.LSH` /
    `SparseAttentionServer`: same method names, same parameter order.
  * `models/attnserver.py` itself drives the two operator classes (`:51-53, 172, 193, 299-300, 329-330`): those calls
    must bind against the mirrors too.
"""
import inspect
import json
import os

import pytest

with open(os.path.join(os.path.dirname(__file__), "golden", "reference_signatures.json")) as _f:
    REF_SIG = json.load(_f)

# reference entry points deliberately not mirrored, with the SURVEY.md row that scopes them out
EXCLUDED = {
    "full_attention": "K=0 dense CPU baseline (SURVEY 2 #2/#5: out of scope; dense layers use attend_dense_kernel)",
    "get_score": "debug view of the fp32 score scratch (sparse_attention.cc:1236-1241); the fused kernel never materialises it",
}


def _bind_call(sig: inspect.Signature, call: dict, bound_method: bool):
    """Replay a reference call (positional count + keyword names) on a mirror signature."""
    args = [object()] * call["nargs"]
    kwargs = {k: object() for k in call["keywords"] if k is not None}
    assert None not in call["keywords"], "reference call uses **kwargs"
    if not bound_method:
        args = [object()] + args  # self
    sig.bind(*args, **kwargs)  # raises TypeError on any mismatch


def test_attnserver_class_signature():
    from magicpig_b200.attnserver import LSHSparseAttnServer as Ours

    ref = REF_SIG["attnserver_methods"]
    assert set(ref) == {"__init__", "alloc_buffer", "fill", "build_table", "plan", "decode", "clear"}
    for name, fn in ref.items():
        assert hasattr(Ours, name), f"mirror lacks method {name}"
        ours = list(inspect.signature(getattr(Ours, name)).parameters.values())
        theirs = fn["args"]
        # same names in the same positions (the mirror may append extra keywords after the reference's)
        assert [p.name for p in ours[: len(theirs)]] == theirs, (name, theirs, [p.name for p in ours])
        # defaults of the reference constructor carry over literally
        for dflt in fn["defaults"]:
            p = next(p for p in ours if p.name == dflt["arg"])
            assert p.default is not inspect.Parameter.empty, f"{name}({dflt['arg']}) lost its default"
            if not dflt["literal"]:
                continue  # torch.bfloat16
            got = list(p.default) if isinstance(p.default, tuple) else p.default
            assert got == dflt["value"], (name, dflt["arg"], got, dflt["value"])
        # anything the mirror adds must be optional
        for p in ours[len(theirs):]:
            assert p.default is not inspect.Parameter.empty, f"{name}: extra parameter {p.name} has no default"


def test_llama_call_sites_bind():
    from magicpig_b200.attnserver import LSHSparseAttnServer as Ours

    seen = set()
    for call in REF_SIG["llama_calls"]:
        name = call["method"]                                                            # __init__: llama.py:92-93
        assert hasattr(Ours, name), f"llama.py calls attention_server.{name}"
        _bind_call(inspect.signature(getattr(Ours, name)), call, bound_method=False)
        seen.add(name)
    assert seen == {"__init__", "decode", "build_table", "fill", "plan", "alloc_buffer", "clear"}, seen


@pytest.mark.parametrize("cc,hdr,cls", [
    ("library/lsh/lsh.cc", "library/lsh/lsh.h", "LSH"),
    ("library/sparse_attention/sparse_attention.cc", "library/sparse_attention/sparse_attention.h", "SparseAttentionServer"),
])
def test_operator_mirrors_cover_pybind_surface(cc, hdr, cls):
    from magicpig_b200 import ops

    Ours = getattr(ops, cls)
    defs = REF_SIG["pybind"][cls]["defs"]           # the .def list of `cc`
    members = REF_SIG["pybind"][cls]["members"]     # the member declarations of `hdr`
    assert len(defs) >= 7
    for name in defs:
        if name in EXCLUDED:
            assert not hasattr(Ours, name), f"{name} is listed as excluded but exists"
            continue
        assert hasattr(Ours, name), f"ops.{cls} lacks the bound method {name}"
        theirs = members[name]
        ours = [p for p in inspect.signature(getattr(Ours, name)).parameters if p != "self"]
        assert ours[: len(theirs)] == theirs, (cls, name, ours, theirs)


def test_attnserver_operator_calls_bind():
    """The reference class drives lsh.LSH / SparseAttentionServer (attnserver.py:51-53,172,193,299-300,329-330); the same
    calls must bind on the mirrors."""
    from magicpig_b200 import ops

    owner = {"attn_server": ops.SparseAttentionServer, "lsh_retriever": ops.LSH}
    n = 0
    for call in REF_SIG["attnserver_operator_calls"]:
        Ours = owner[call["owner"]]
        assert hasattr(Ours, call["method"]), (call["owner"], call["method"])
        _bind_call(inspect.signature(getattr(Ours, call["method"])), call, bound_method=False)
        n += 1
    assert n >= 7, n


def test_stored_signatures_match_reference_sources():
    """The stored surface is what the reference's sources say, wherever a reference checkout is readable."""
    from oracle.build_ref import REF
    if not os.path.isfile(os.path.join(REF, "models", "attnserver.py")):
        pytest.skip("no readable reference checkout (MAGICPIG_REFERENCE)")
    from tests.golden.make_golden import reference_signatures
    assert json.loads(json.dumps(reference_signatures(REF))) == REF_SIG
