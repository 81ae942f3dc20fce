"""groth16_b200 -- H100-native (sm_90a) Groth16 proving hot path: NTT witness map + five MSMs behind the
ark-groth16 `create_proof_with_reduction_and_matrices` interface.  See DESIGN.md / INTEGRATION.md."""
import os as _os

# A proof runs on 6 CUDA streams per slot; with the default 8 hardware work queues streams share queues and serialise
# behind each other (csrc/api.cu, g16_ctx_create).  Read when the CUDA context is created: set it before anything touches
# the device.  An explicit user setting wins.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from .api import (ConstraintMatrices, CudaError, Groth16, MalformedKey, PolynomialDegreeTooLarge, Proof, ProvingKey,
                  SynthesisError, VerifyingKey)
from .codec import CurveCodec, FieldCodec
from .params import BLS12_377, BLS12_381, BN254, CURVES, get_curve

__all__ = ["Groth16", "ConstraintMatrices", "ProvingKey", "VerifyingKey", "Proof", "SynthesisError",
           "PolynomialDegreeTooLarge", "MalformedKey", "CudaError", "CurveCodec", "FieldCodec", "CURVES", "BLS12_381",
           "BN254", "BLS12_377", "get_curve"]
