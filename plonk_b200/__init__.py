"""plonk_b200 - H100-native backend for the dusk-plonk prover hot path (NTT + G1 MSM).

Host-side mirror of the reference's crate-private seam (SURVEY.md section 8b):

    EvaluationDomain.{fft, ifft, coset_fft, coset_ifft}   reference src/fft/domain.rs:166-232
    CommitKey.commit                                      reference src/commitment_scheme/kzg10/key.rs:376-388
    PublicParameters.setup / from_slice                   reference src/commitment_scheme/kzg10/srs.rs:61-178
    DevicePublicParameters                                the same, resident on the GPU and shared by the provers
                                                          compiled from it
    Compiler.compile / compile_with_circuit               reference src/compiler.rs:116-461
    Compiler.compile_with_compressed, compress            reference src/compiler.rs:84-112, src/composer/circuit.rs:28-45
    unsatisfied_constraints / unsatisfied_report,         reference src/debugger.rs:95-236
      Prover.unsatisfied_constraints / _report

Everything computes on the GPU through the C ABI in include/plonk_b200.h; there is no CPU path."""
from ._lib import Pb200Error, PlonkVersion, lib  # noqa: F401
from .debugger import identity_family, unsatisfied_constraints, unsatisfied_report  # noqa: F401
from .compiler import BlsScalarMalformed, Compiler, InvalidCompressedCircuit, TruncatedDegreeTooLarge, compress, compress_arrays  # noqa: F401
from .domain import EvaluationDomain  # noqa: F401
from .kzg import CommitKey, Commitment, PolynomialDegreeTooLarge  # noqa: F401
from .prover import CircuitUnsatisfied, Prover, UnsupportedProvingVersion  # noqa: F401
from .srs import DegreeIsZero, DevicePublicParameters, NotEnoughBytes, PublicParameters, PublicParameterTables  # noqa: F401
from .verifier import PointMalformed, ProofVerificationError, Verifier, batch_verify_groups  # noqa: F401
