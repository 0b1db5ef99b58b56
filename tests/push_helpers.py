"""Shared by the tests of the update kernels (push kernel, mailbox applier) and of the push paths of the training step."""
import time

# every optimizer configuration the update kernels are checked with: all ten rules, Nesterov momentum and centered RMSProp
OPTIMIZERS = [
    ("gradient_descent", dict(learning_rate=0.1)),
    ("momentum", dict(learning_rate=0.1, momentum=0.9)),
    ("momentum", dict(learning_rate=0.1, momentum=0.9, use_nesterov=True)),
    ("adam", dict(learning_rate=0.01, beta1=0.85, beta2=0.98, epsilon=1e-8)),
    ("rmsprop", dict(learning_rate=0.05, decay=0.95, momentum=0.1, epsilon=1e-10)),
    ("rmsprop", dict(learning_rate=0.05, decay=0.95, momentum=0.1, epsilon=1e-6, centered=True)),
    ("adagrad", dict(learning_rate=0.1, initial_accumulator_value=0.1)),
    ("adadelta", dict(learning_rate=1.0, rho=0.95, epsilon=1e-6)),
    ("adagrad_da", dict(learning_rate=0.1, l1_regularization_strength=0.001, l2_regularization_strength=0.01)),
    ("ftrl", dict(learning_rate=0.1, l1_regularization_strength=0.001, l2_regularization_strength=0.01)),
    ("proximal_adagrad", dict(learning_rate=0.1, l1_regularization_strength=0.001, l2_regularization_strength=0.01)),
    ("proximal_gradient_descent", dict(learning_rate=0.1, l1_regularization_strength=0.001,
                                       l2_regularization_strength=0.01)),
]


def wait_pushes(master, n, timeout_s=10.0):
    """Poll the master's applied-push counter until it reaches ``n`` (an applier bumps it a few stores after the
    acknowledgement a worker waits for); returns the last value read."""
    t0 = time.time()
    while master.counters()["pushes"] < n and time.time() - t0 < timeout_s:
        time.sleep(0.002)
    return master.counters()["pushes"]
