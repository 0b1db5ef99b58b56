import os
import sys

import pytest

# several workers + appliers share one GPU in the tests: one hardware launch queue per stream (see sparkflow_b200/__init__.py)
os.environ.setdefault("SPARKFLOW_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU of compute capability 9.0 (H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_makereport(item, call):
    outcome = yield
    rep = outcome.get_result()
    if rep.failed and "gpu" in item.keywords:
        try:
            from sparkflow_b200.ops import native

            rep.sections.append(("sparkflow_b200 device error channel", native.describe_device_error()))
        except Exception:
            pass


def pytest_terminal_summary(terminalreporter, exitstatus, config):
    """Which engine actually ran: a GPU run that only exercised the PyTorch interpreter must not look like a native run."""
    try:
        import torch

        if not torch.cuda.is_available():
            return
        from sparkflow_b200.ops import native
        from sparkflow_b200.parallel.session import ENGINE_USES

        ext = native.cuda_ext()
        terminalreporter.write_line(
            "sparkflow_b200 engines used by TrainingSession in this run: "
            + (", ".join(f"{k}={v}" for k, v in sorted(ENGINE_USES.items())) or "none")
            + f"; native extension: {getattr(ext, '__file__', '?')}")
    except Exception as exc:  # pragma: no cover
        terminalreporter.write_line(f"sparkflow_b200 engine summary unavailable: {exc}")


@pytest.fixture(scope="session")
def tf_checkpoint(tmp_path_factory):
    """A self-generated TF-V2 checkpoint of the reference fixture's architecture (2-10 tanh-10 tanh-1 sigmoid, Adam
    slots, beta powers: the key set of tests/golden/test_model/to_load.index) written by this package's own
    bundle writer - the suite does not depend on the reference tree being mounted."""
    import numpy as np

    from sparkflow_b200.graph.executor import GraphProgram
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.models import zoo
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.utils.checkpoint import save_master_state

    d = tmp_path_factory.mktemp("test_model")
    graph = zoo.build("fixture_mlp")
    ir = GraphIR.from_metagraph(graph)
    w = GraphProgram(ir).init_weights(seed=11)
    rng = np.random.default_rng(5)
    slots = [[rng.normal(0, 0.01, a.shape).astype(np.float32) for a in w], [np.abs(rng.normal(0, 0.01, a.shape)).astype(np.float32) for a in w]]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.1))
    prefix = save_master_state(str(d / "to_load"), [v.name for v in ir.trainable], w, slots, spec, step=37, graph_json=graph)
    return dict(prefix=prefix, weights=w, slots=slots, graph=graph)
