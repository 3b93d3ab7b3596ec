import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
	sys.path.insert(0, ROOT)


def pytest_configure(config):
	config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built_library():
	"""The CUDA library must exist; tests never fall back to a CPU path."""
	from vulkan_renderer_b200 import api
	if not os.path.exists(api.LIB_PATH):
		import __graft_entry__
		__graft_entry__.build_library()
	return api.load_library()
