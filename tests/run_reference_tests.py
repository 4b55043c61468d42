"""Run the REFERENCE's own hot-path unit tests against THIS implementation.

The reference's package, byte-compiled by oracle/build_ref.py into oracle/_ref/reftests,
supplies the test modules and their helpers (local master, fixtures); the
flash-checkpoint modules they import —
dlrover.python.common.{multi_process,storage,...},
dlrover.python.elastic_agent.torch.ckpt_saver,
dlrover.trainer.torch.flash_checkpoint.* — are replaced by this package's
modules before the tests are loaded (dlrover_b200.compat.ALIASES, real parent
packages kept).  The modules are sourceless, so unittest (all of them are
unittest.TestCase suites) runs them, not pytest.  Usage:

    python tests/run_reference_tests.py [test module or reference-relative path ...]
"""

import importlib
import os
import sys
import tempfile
import unittest
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "reftests")

DEFAULT_FILES = [
    "dlrover/python/tests/test_multi_process.py",
    "dlrover/python/tests/test_storage.py",
    "dlrover/python/tests/test_ckpt_saver.py",
    "dlrover/trainer/tests/torch/checkpoint_egine_test.py",
    "dlrover/trainer/tests/torch/ddp_checkpointer_test.py",
    "dlrover/trainer/tests/torch/megatron_ckpt_test.py",
    "dlrover/trainer/tests/torch/checkpoint_backup_test.py",
    "dlrover/trainer/tests/torch/fsdp_ckpt_test.py",
]


class _StubFinder:
    """`import kubernetes[.anything]` -> MagicMock modules (the package is not in
    this image; the reference's test helpers import it at module level)."""

    PREFIXES = ("kubernetes",)

    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in self.PREFIXES:
            import importlib.machinery

            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = mock.MagicMock()
        m.__name__ = spec.name
        m.__path__ = []
        m.__spec__ = spec
        return m

    def exec_module(self, module):
        pass


def install_overrides():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    sys.meta_path.insert(0, _StubFinder())
    os.environ.setdefault("ROLE_NAME", "dlrover-trainer")
    os.environ.setdefault("DLROVER_B200_ASYNC_DRAIN", "0")  # the tests assume blocking saves
    from dlrover_b200 import compat

    # constants/log/env_utils stay the reference's (the test helpers need the
    # full modules); the path under test is swapped
    keep_real = {"dlrover.python.common.constants", "dlrover.python.common.log",
                 "dlrover.python.common.env_utils", "dlrover.python.common.singleton",
                 "dlrover.python.common.serialize"}
    swapped = []
    for alias, target in compat.ALIASES.items():
        if alias in keep_real:
            continue
        parent = alias.rsplit(".", 1)[0]
        importlib.import_module(parent)  # the real package
        mod = importlib.import_module(target)
        sys.modules[alias] = mod
        setattr(sys.modules[parent], alias.rsplit(".", 1)[1], mod)
        swapped.append(alias)
    return swapped


if __name__ == "__main__":
    # children started by the tests (mp.spawn) get the overrides through
    # tests/_ref_site/sitecustomize.py
    os.environ["DLROVER_B200_REF_TESTS"] = "1"
    # the reference's event exporter logs to /tmp/dlrover by default, a directory that may
    # belong to another user: every run gets its own (inherited by spawned children)
    work = tempfile.mkdtemp(prefix="fc_reftests_")
    os.environ["DLROVER_EVENT_FILE_DIR"] = os.path.join(work, "events")
    site = os.path.join(ROOT, "tests", "_ref_site")
    os.environ["PYTHONPATH"] = os.pathsep.join(
        [site, ROOT, REF] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p])
    sys._fc_ref_overrides = True
    swapped = install_overrides()
    print(f"[run_reference_tests] {len(swapped)} reference modules replaced by dlrover_b200")
    names = [a[:-3].replace("/", ".") if a.endswith(".py") else a
             for a in (sys.argv[1:] or DEFAULT_FILES)]
    os.chdir(work)
    suite = unittest.defaultTestLoader.loadTestsFromNames(names)
    result = unittest.TextTestRunner(verbosity=2).run(suite)
    failed = len(result.failures) + len(result.errors) + len(result.unexpectedSuccesses)
    passed = result.testsRun - failed - len(result.skipped) - len(result.expectedFailures)
    print(f"{passed} passed" + (f", {failed} failed" if failed else "")
          + (f", {len(result.skipped)} skipped" if result.skipped else ""), flush=True)
    sys.exit(0 if failed == 0 else 1)
