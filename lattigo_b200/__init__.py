"""lattigo_b200 -- H100-native (sm_90a) RNS polynomial-ring engine behind Lattigo's `ring` /
`rlwe.Evaluator` hot-path interface. The compute lives in csrc/ (hand-written CUDA + C ABI,
include/lattigo_b200.h); this package is the thin host-side mirror of the reference's method names
used by the tests and the benchmark. No CPU fallback exists."""
from ._lib import LgpuError, lib, declared_symbols, SO_PATH  # noqa: F401
from .ring import Context, Ring, SubRing, OPS, OP  # noqa: F401
from .rlwe import (GadgetCiphertext, BasisExtender, Decomposer, Evaluator, CKKSEvaluator, div_by_last_modulus_many,  # noqa: F401
                   automorphism_ntt_index, automorphism_ntt_with_index, automorphism_ntt, automorphism)
from .ringqp import RingQP, Poly as PolyQP  # noqa: F401
from .bgv import BGVEvaluator  # noqa: F401
from . import lintrans  # noqa: F401,E402
from . import innersum  # noqa: F401,E402
from . import ringpacking  # noqa: F401,E402
from . import wire  # noqa: F401,E402
from . import rgsw  # noqa: F401,E402
from . import encryptor  # noqa: F401,E402
from . import multiparty  # noqa: F401,E402
from . import mpbgv  # noqa: F401,E402
from . import mpckks  # noqa: F401,E402
from . import ckks_fft  # noqa: F401,E402
from .encoder import Encoder  # noqa: F401,E402
from .bgv_encoder import BGVEncoder  # noqa: F401,E402
from .bgv_polyeval import BGVPolynomialEvaluator  # noqa: F401,E402
