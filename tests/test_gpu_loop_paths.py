"""The iteration graph's loop body against the host launch loop.

test_gpu_parity.py::test_graph_loop_equals_host_loop compares use_graph = 1 with use_graph = 0 on a small batch, which
the cooperative kernel takes (DESIGN §4.3). Here the batches are ones the cooperative kernel never takes, so that
use_graph = 1 runs the recorded WHILE body: three C2 pairs resident on one context (about 2,800 source chunks, more
than the 16 blocks x 132 SMs the cooperative kernel can hold on an H100), and a pair with normal shooting. Both loop
implementations must give bit-identical results and traces."""
import numpy as np
import pytest

from mulls_b200 import abi, synth

pytestmark = pytest.mark.gpu


def test_graph_body_equals_host_loop(small_pair):
    from mulls_b200.registration import Context

    shoot = abi.IcpParams.from_buffer_copy(small_pair["params"])
    shoot.normal_shooting_on = 1
    batches = {"c2 x3": [synth.make_pair(s, "c2") for s in (1001, 1005, 1006)],
               "normal shooting": [dict(small_pair, params=shoot)]}
    for name, batch in batches.items():
        n_src = max(sum(len(c) for c in q["src"]) for q in batch)
        n_tgt = max(sum(len(c) for c in q["tgt"]) for q in batch)
        out = {}
        for mode in (1, 0):
            ctx = Context(0, len(batch), n_src, n_tgt)
            ctx.set_tunable("use_graph", mode)
            ctx.upload(batch)  # the whole batch on this one context (a one-shot batch is split over it and its twin)
            out[mode] = ctx.run_resident(want_trace=True)
            if mode == 1:  # the graph ran: six kernels per iteration, not one cooperative launch
                assert ctx.stats()["kernel_launches"] >= 6 * max(r["iters"] for r in out[mode][0])
            again = ctx.run_resident(want_trace=True)  # the recorded graph is re-launched, not rebuilt
            for a, b in zip(out[mode][0], again[0]):
                assert np.array_equal(a["T"], b["T"]) and a["iters"] == b["iters"]
            ctx.close()
        for (a, ta), (b, tb) in zip(zip(*out[1]), zip(*out[0])):
            for r, s in ((a, b), (ta, tb)):
                assert r.keys() == s.keys()
                for k in r:
                    np.testing.assert_array_equal(r[k], s[k], err_msg=f"{name}: {k}")
            assert ta["n_iter"] >= 1
