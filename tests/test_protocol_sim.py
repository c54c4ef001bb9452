"""The context-parallel exchange protocol of the attention kernel (ready words, buffer parity, exit wait;
tools/sim_cp_protocol.py) checked by discrete-event simulation: ranks at random relative speeds must neither deadlock
nor read a buffer that is not ready.  Runs in a few seconds on the CPU."""
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cp():
    spec = importlib.util.spec_from_file_location("sim_cp", os.path.join(ROOT, "tools", "sim_cp_protocol.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_context_parallel_buffer_reuse_protocol_needs_no_barrier_between_layers():
    """Ready words + buffer parity + exit wait (DESIGN.md section 5): ranks at arbitrary relative speeds, 6 layers."""
    sim = _cp()
    for seed in range(60):
        for cp in (2, 4, 8):
            sim.Sim(cp, 6, seed).run()


def test_context_parallel_simulator_sees_a_broken_protocol():
    sim = _cp()

    class Sparse(sim.Sim):                   # a read pattern in which a rank does not hear from every peer by reading
        def reads_from(self, r):
            return [(r + 1) % self.cp]

    def failures(cls, variant, cp=4):
        n = 0
        for seed in range(40):
            try:
                cls(cp, 6, seed, variant=variant).run()
            except (AssertionError, RuntimeError):
                n += 1
        return n

    assert failures(sim.Sim, "no_ready_wait") > 0          # reading before the owner announced its rows
    assert failures(sim.Sim, "flag_before_write") > 0      # announcing before the rows are written
    assert failures(Sparse, "") == 0                       # the full protocol does not depend on the read pattern ...
    assert failures(Sparse, "no_exit_wait") > 0            # ... because of the exit wait
