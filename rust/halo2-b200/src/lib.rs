//! `halo2_proofs_axiom_gpu`: what halo2-lib sees as `halo2_proofs` under its `cuda` feature
//! (halo2-base/src/lib.rs:25-28).  The fork of halo2-axiom 0.5.3 keeps every public path halo2-lib
//! imports (SURVEY.md §8(b) lists them) and replaces four bodies with calls into [`backend`]:
//!
//! | halo2-axiom function                                   | becomes                                   |
//! |--------------------------------------------------------|-------------------------------------------|
//! | `ParamsKZG::{commit, commit_lagrange}`                 | [`backend::Backend::commit`]              |
//! | `arithmetic::best_fft`, `EvaluationDomain::*`          | [`backend::Backend::best_fft`] and friends |
//! | `WitnessCollection` filled by halo2-base `assign_witnesses` | [`backend::Backend::assign_witnesses`] |
//! | `evaluate_h`, product columns, openings                | the `_dev` entry points on [`backend::Poly`] handles |
//!
//! No exception or abort crosses the boundary: every C entry point returns a status; [`backend::check`] turns a
//! non-zero status into the panic the CPU path raises (`.expect("prover should not fail")`,
//! halo2-base/src/utils/testing.rs:48), which is safe under `panic = "unwind"` (reference Cargo.toml:31).
pub mod backend;
pub mod ffi;
