"""mega_core -- H100-native drop-in for the inference hot path of Scalsol/mega.pytorch.

Mirrors the reference's `mega_core` operator / module API for that path (see INTEGRATION.md);
every compute op is a hand-written sm_90a kernel behind libmega_b200.so.
"""
