"""The brick face-list prototype (tools/brick_face_lists.py): its build-time cull, a bound meant to hold for every point
of a brick, must keep each lattice point's brute-force nearest face and every face that ties with it."""
from tools import brick_face_lists as B


def test_face_lists_keep_every_nearest_face():
    r = B.run(bricks_n=4, near_n=4, seed=1)
    c = r["conservative"]
    assert c["points"] == 8 * r["warps_per_brick"] * 32
    assert c["nearest_not_listed"] == 0
    assert c["left_out_ties"] == 0
    assert r["near_body"]["bricks"] == 4
    # the lists only drop faces of today's leaf lists
    assert r["uniform"]["face_list_len"]["mean"] <= r["uniform"]["leaf_list_faces"]["mean"]
