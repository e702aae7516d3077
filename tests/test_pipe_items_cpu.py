"""CPU: the plan-cache records of 64-pixel work items.  The cache keeps one 32-pixel record slot per 32-pixel tile (plus the tail
halves), and its size is pinned per shape; a 64-pixel claim c takes slots 2c and 2c + 1.  This restates the kernel's claim count
(whole tiles + the split last round) and checks that, on every shape that runs 64-pixel items, every claim's two slots lie inside
the region, so no claim falls back to rebuilding its item each call."""
import itertools


def records(N, n_ref, H, W):                     # fusion_pipe_plan_records
    return N * -(-H * W // 32) + (N // n_ref) * (256 + n_ref)


def claims(N, n_ref, H, W, sms, P):
    tpi = -(-H * W // P)
    grid = min(N * tpi, sms)
    grid1 = min(n_ref * tpi, grid)
    tail = (n_ref * tpi) % grid1
    r_half = 0 if P == 64 and 2 * tail > grid1 else min(tpi, -(-tail // n_ref))
    return N * (tpi - r_half) + 2 * N * r_half


def test_plan_record_slots_hold_every_64_pixel_claim():
    for H, W, n_ref, S, sms in itertools.product(range(2, 65, 3), range(2, 65, 5), (1, 2, 3, 4, 8, 64), (1, 2, 3), (132, 114, 66, 7)):
        N = S * n_ref
        assert 2 * claims(N, n_ref, H, W, sms, 64) <= records(N, n_ref, H, W), (H, W, n_ref, S, sms)

