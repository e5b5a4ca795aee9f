"""Import-path shim: `datasets.*` as the reference scripts spell it.  Synthetic stand-ins are provided for
`datasets.audioset`, `datasets.esc50`, `datasets.dcase20`, `datasets.fsd50k` and `datasets.openmic` (see each module);
anything else keeps importing from the reference checkout."""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
