"""Drop-in shim: put `<repo>/compat` in front of the reference checkout on `sys.path` and the reference's own programs
(`tools/test_reconstruction_hf.py:37-39`, `tools/test_zero_shot_hf.py:38-39`, `generation/tokenizer/vtp_tokenizer.py:6`)
import the H100 implementation through their unchanged `from vtp.models.vtp_hf import VTPModel` lines.

Only the hot path is replaced (SURVEY.md §8b): `vtp.models.vtp_hf`.  Everything else those programs import from the
`vtp` package (`vtp.tokenizers`, `vtp.utils.*`) is out of scope and resolves to the reference checkout when it is on the
path — this package extends its search path over every other `vtp/` directory instead of copying those modules."""
import pkgutil

__path__ = pkgutil.extend_path(__path__, __name__)
