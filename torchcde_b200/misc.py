"""The reference's ``torchcde.misc`` names (misc.py:70-166)."""
from .coeffs import forward_fill, validate_input_path
from .controls import TupleControl

__all__ = ["forward_fill", "validate_input_path", "TupleControl"]
