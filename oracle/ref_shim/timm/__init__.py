"""Five-symbol stand-in for `timm` (not installed, no network) so that the UNMODIFIED reference
package can be imported by oracle/make_golden.py without timm installed.
Test infrastructure only — never imported by the product path. Semantics restated from timm 0.9.6
(the version the reference pins, requirements.txt:1)."""
