"""lib.psa.functional of the reference (lib/psa/functional.py:4-5) on the sm_90a kernel; no JIT build at import."""
from semseg_b200.psa import psa_mask  # noqa: F401
