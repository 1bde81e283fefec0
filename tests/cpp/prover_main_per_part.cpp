// prover_main with a per-part proving key (Cosets::PerPart): the same program as prover_main.cpp, whose one keygen call is
// redirected here to the per-part mode, so both binaries read the same dumped case and must write the same proof bytes.
#ifdef SPB_PROVER_WITH_CUDART
#include <cuda_runtime.h>
#endif
#include "../../include/spectre_b200_prover.hpp"

#define keygen(E, cs, fixed, copies, digest) keygen(E, cs, fixed, copies, digest, halo2::plonk::Cosets::PerPart)
#include "prover_main.cpp"
