"""halo2-lib_b200 — host-side mirror (Python, for tests / bench plumbing) of the prover interfaces that the
H100 back end implements behind the C ABI of include/h2b200.h.  The C++ mirror for a compiled host is
include/h2b200.hpp; the Rust binding a maintainer adds is shown in INTEGRATION.md."""
from ._capi import lib, LIB_PATH, SIGNATURES, header_symbols, H2B_ERR_ARG, CHECK_MAX_REPORT  # noqa: F401
from .parallel import shard_range, ntt_owner, ntt_owners_balanced, all_gather_points, connect_peers, allreduce_points  # noqa: F401
from .host import (  # noqa: F401
    H2BError,
    LayoutError,
    ConstraintSystemFailure,
    Context,
    ParamsKZG,
    gen_srs,
    srs_path,
    seeded_tau,
    g2_generator_mul,
    EvaluationDomain,
    best_multiexp,
    best_fft,
    assign_witnesses,
    assign_witnesses_assigned,
    assign_lookups,
    apply_rational_dev,
    assign_lookups_indexed_dev,
    omega,
)
from .evaluation import (  # noqa: F401,E402
    GraphEvaluator,
    BoundGraph,
    quotient_graph,
    permutation_fold,
    lookup_fold,
    divide_by_vanishing_poly,
    eval_polynomial,
    kate_division,
    poly_lincomb,
    permute_expression_pair,
)
from .prover import Poly, Circuit, ProverSession, MockProver, keygen, synthetic_circuit  # noqa: F401,E402
