"""The column-major search kernels leave the displaced lists of the base they end on in HBM themselves (CTA 0 stores its
shared-memory copy after the last round); no list rebuild runs after them.  The row-major per-round kernel reads those
lists, so its keys on the searched session must be the restatement's on the same base, also when patience stops the
search before its last round."""
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m
from problems import moved_base
from test_gpu_large_layouts import assert_keys

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(1000, 64, 8, 3, 0), (256, 32, 4, 3, 2)])
def test_row_major_round_reads_the_lists_a_column_major_search_left(ref_lib, shape):
    pb = m.synthetic_problem(*shape)
    r = ref_lib.Ref(pb)
    start = moved_base(pb, r.decode(*r.init_base()), 6)
    seed, size, ksize = 0x11575, 512, 2048
    for patience, rounds in ((0, 7), (4, 3000)):
        sess = kao.Session(kao.Problem.from_fields(pb))
        assert sess.stats()["column_major"]
        sess.set_base(start)
        sess.set_patience(patience)
        keys, _ = sess.search(seed, 0, rounds, size)
        ran = sess.last_rounds()
        assert 0 < ran <= rounds and (patience == 0) == (ran == rounds)
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, seed, 0, ran, size)
        assert_keys(keys[:ran], want, ("search", patience))
        reps, _, _, _ = sess.get_base()
        assert (reps == r.decode(bits, ld)).all()
        want_next = r.candidate_keys(bits, ld, seed, ran, ksize, 0, ksize)
        assert sess.set_evaluator(False)
        assert_keys(sess.candidate_keys(seed, ran, ksize, 0, ksize), want_next, ("row-major round", patience))
        sess.close()
