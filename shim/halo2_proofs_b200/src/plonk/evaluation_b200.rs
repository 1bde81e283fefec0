//! `GraphEvaluator` -> `spb_graph`: the flat program `spb_graph_evaluate_dev` interprets for every extended row
//! ([UPSTREAM] halo2_proofs/src/plonk/evaluation.rs: `GraphEvaluator { constants, rotations, calculations,
//! num_intermediates }`, `Calculation`, `ValueSource`; `Evaluator::evaluate_h` is stage 8 of create_proof, reached from
//! Spectre at lightclient-circuits/src/util/circuit.rs:158,211).
//!
//! Encoding (include/spectre_b200.h, `spb_graph`), all little-endian u32 words:
//!   per calculation: word0 = op | nparts << 8, word1 = target intermediate, then two words per source: (kind, idx | rot_idx << 16)
//!   op:   0 Add  1 Sub  2 Mul  3 Square  4 Double  5 Negate  6 Horner  7 Store
//!   kind: 0 Constant 1 Intermediate 2 Fixed 3 Advice 4 Instance 5 Challenge 6 Beta 7 Gamma 8 Theta 9 Y 10 PreviousValue
//!   Add / Sub / Mul: a, b.   Square / Double / Negate / Store: a.   Horner: start value, factor, then the `nparts` parts.
//! The interpreter is `graph_evaluate_row` in spectre_b200/csrc/quotient.cuh; tests/test_gpu_quotient.py and
//! tests/test_hostemu_quotient.py check it against a CPU restatement of `GraphEvaluator::evaluate` on random gate graphs.
//!
//! `Evaluator` gets one cached `FlatGraph` per `GraphEvaluator` it owns (custom gates; per lookup the compressed input /
//! table expressions), built once in `Evaluator::new` -- patches/evaluation.patch.

use super::evaluation::{Calculation, GraphEvaluator, ValueSource};
use crate::b200::spb_graph;
use halo2curves::bn256::{Fr, G1Affine};

pub struct FlatGraph {
    pub program: Vec<u32>,
    pub num_calculations: u32,
    pub num_intermediates: u32,
    pub constants: Vec<Fr>,
    pub rotations: Vec<i32>,
}

fn src(v: &ValueSource) -> [u32; 2] {
    // (kind, idx | rot_idx << 16); the index fields are 16 bits wide -- checked in `flatten`
    match *v {
        ValueSource::Constant(i) => [0, i as u32],
        ValueSource::Intermediate(i) => [1, i as u32],
        ValueSource::Fixed(col, rot) => [2, col as u32 | (rot as u32) << 16],
        ValueSource::Advice(col, rot) => [3, col as u32 | (rot as u32) << 16],
        ValueSource::Instance(col, rot) => [4, col as u32 | (rot as u32) << 16],
        ValueSource::Challenge(i) => [5, i as u32],
        ValueSource::Beta() => [6, 0],
        ValueSource::Gamma() => [7, 0],
        ValueSource::Theta() => [8, 0],
        ValueSource::Y() => [9, 0],
        ValueSource::PreviousValue() => [10, 0],
    }
}

/// Flatten one evaluator. Returns `None` when an index does not fit the 16-bit fields (the caller then keeps the CPU loop
/// for this evaluator; halo2-lib / zkevm-hashes circuits are far below the limit: a few hundred calculations).
pub fn flatten(ev: &GraphEvaluator<G1Affine>) -> Option<FlatGraph> {
    if ev.num_intermediates > 0xffff || ev.constants.len() > 0x1_0000 || ev.rotations.len() > 0xffff {
        return None;
    }
    let mut p = Vec::<u32>::with_capacity(ev.calculations.len() * 6);
    for info in &ev.calculations {
        let mut emit = |op: u32, nparts: u32, srcs: &[&ValueSource]| {
            p.push(op | nparts << 8);
            p.push(info.target as u32);
            for s in srcs {
                p.extend_from_slice(&src(s));
            }
        };
        match &info.calculation {
            Calculation::Add(a, b) => emit(0, 0, &[a, b]),
            Calculation::Sub(a, b) => emit(1, 0, &[a, b]),
            Calculation::Mul(a, b) => emit(2, 0, &[a, b]),
            Calculation::Square(a) => emit(3, 0, &[a]),
            Calculation::Double(a) => emit(4, 0, &[a]),
            Calculation::Negate(a) => emit(5, 0, &[a]),
            Calculation::Horner(start, parts, factor) => {
                if parts.len() > 0xff_ffff {
                    return None;
                }
                let mut s: Vec<&ValueSource> = vec![start, factor];
                s.extend(parts.iter());
                emit(6, parts.len() as u32, &s)
            }
            Calculation::Store(a) => emit(7, 0, &[a]),
        }
    }
    Some(FlatGraph {
        program: p,
        num_calculations: ev.calculations.len() as u32,
        num_intermediates: ev.num_intermediates as u32,
        constants: ev.constants.clone(),
        rotations: ev.rotations.clone(),
    })
}

impl FlatGraph {
    /// the C view; valid while `self` is alive
    pub fn as_spb(&self) -> spb_graph {
        spb_graph {
            program: self.program.as_ptr(),
            program_words: self.program.len(),
            num_calculations: self.num_calculations,
            num_intermediates: self.num_intermediates,
            constants: self.constants.as_ptr(),
            num_constants: self.constants.len() as u32,
            rotations: self.rotations.as_ptr(),
            num_rotations: self.rotations.len() as u32,
        }
    }
}

// What `Evaluator::evaluate_h` becomes with the device-resident pipeline (per circuit instance; all pointers are device
// buffers of 2^extended_k rows produced by spb_coeff_to_extended_batch_dev; `values` starts zeroed):
//
//   spb_graph_evaluate_dev(ctx, &custom_gates.as_spb(), fixed_cosets, advice_cosets, instance_cosets, challenges,
//                          beta, gamma, theta, y, values, size, rot_scale);                 // GraphEvaluator over every row
//   spb_permutation_constraints_dev(ctx, values, size, rot_scale, last_rotation, n_sets, chunk_len, z_cosets, n_cols,
//                          column_cosets, sigma_cosets, l0, l_last, l_active, beta, gamma, y, extended_omega);
//   for each lookup:
//       spb_graph_evaluate_dev(ctx, &lookup_value_graph.as_spb(), ..., table_value, size, rot_scale);   // (a + beta)(s + gamma)
//       spb_lookup_constraints_dev(ctx, values, size, rot_scale, product_coset, permuted_input_coset, permuted_table_coset,
//                          table_value, l0, l_last, l_active, beta, gamma, y);
//
// -- the same sequence as spectre_b200/plonk.py::create_proof stage 7 and include/spectre_b200_prover.hpp, whose proofs
// the reference's verifier contracts accept (DESIGN.md section 2). On a context with several devices each of these
// passes is split into row ranges across the devices by the library; nothing changes on this side.
// With a lean proving key (INTEGRATION.md section 4, "Key residency") fixed_cosets, sigma_cosets and l0 / l_last / l_active
// are not held by the key: they are rebuilt from the key's coefficient forms by one spb_coeff_to_extended_batch_dev call
// just before this sequence and freed after it, before divide_by_vanishing. The sequence itself does not change.
