"""mmsr-compatible package surface of the H100 build.

Keeps the reference's arch/model registry and options-YAML API (SURVEY.md §8b B3) so
`python mmsr/test.py -opt options/test/test_C2_matching_mse.yml` and reference checkpoints work
unchanged, while the restoration-forward hot path runs in libc2m_sm100.so."""
__version__ = '0.1.0+b200'
