"""cluster-capacity_b200 — H100-native hot path of kubernetes-sigs/cluster-capacity (see DESIGN.md).

The directory name contains a hyphen (it is the name the build contract asks for), so import it with
`importlib.import_module("cluster-capacity_b200")`.
"""
from . import _abi as abi  # noqa: F401
