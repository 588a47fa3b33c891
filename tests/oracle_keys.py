"""TEST INFRASTRUCTURE: OracleEnv with a switchable Philox key (tests/oracle_keys.c).

The shim is compiled with the oracle's compiler flags into a temporary directory (keyed by a hash of its sources), so
the tree is never written. Its oracle_set_key writes the key of an env created through oracle/binding.py.
"""

import ctypes
import hashlib
import os
import subprocess
import tempfile

from oracle import binding

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SOURCES = (os.path.join(_HERE, 'oracle_keys.c'), os.path.join(_ROOT, 'oracle', 'mp_oracle.c'),
            os.path.join(_ROOT, 'include', 'mpb_format.h'))
_lib = None


def lib() -> ctypes.CDLL:
  global _lib
  if _lib is None:
    digest = hashlib.sha256(b''.join(open(p, 'rb').read() for p in _SOURCES)).hexdigest()[:16]
    path = os.path.join(tempfile.gettempdir(), f'mp_oracle_keys_{os.getuid()}_{digest}.so')
    if not os.path.exists(path):
      tmp = f'{path}.{os.getpid()}'
      subprocess.check_call(['gcc', '-O2', '-fPIC', '-shared', '-ffp-contract=off', '-std=c11', '-w', '-o', tmp,
                             _SOURCES[0], '-lm', '-lpthread'])
      os.replace(tmp, path)
    L = ctypes.CDLL(path)
    L.oracle_set_key.argtypes = [ctypes.c_void_p, ctypes.c_uint64]
    _lib = L
  return _lib


class KeyedOracleEnv(binding.OracleEnv):
  """An OracleEnv whose Philox key can be switched (oracle_set_key)."""

  def set_key(self, key: int) -> None:
    """Every later draw of this env uses `key`, as a restore with MP_RESTORE_REKEY gives the restored env its own."""
    lib().oracle_set_key(self._h, ctypes.c_uint64(int(key)))
