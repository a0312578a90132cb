"""tests/kernel_census.py on literal demangled kernel names, without a GPU."""
import kernel_census


def items(*names):
    return kernel_census.variants([(n, 1) for n in names])


def test_profiler_names_keep_their_template_arguments():
    for raw, name in [("void sbn_step_batched<8, 0, SbnLogSumExp>(SbnStep)", "sbn_step_batched<8, 0, SbnLogSumExp>"),
                      ("void sbn_step_flat<float, SbnMaxSum>(SbnStep)", "sbn_step_flat<float, SbnMaxSum>"),
                      ("sbn_argmax_step(SbnSample)", "sbn_argmax_step"),
                      ("void sbn_step_batched<2, 4>(SbnStep)", "sbn_step_batched<2, 4>")]:
        m = kernel_census._KERNEL.search(raw)
        assert m.group(1) + (f"<{m.group(2)}>" if m.group(2) is not None else "") == name


def test_policy_instantiations_get_items_of_their_own():
    for n in range(1, 9):
        assert items(f"sbn_step_batched<{n}, 0, SbnMaxSum>") == {f"batched N_IN={n} SbnMaxSum"}
        assert items(f"sbn_step_batched<{n}, 0, SbnLogSumExp>") == {f"batched N_IN={n} SbnLogSumExp"}
    assert items("sbn_step_flat<float, SbnMaxSum>") == {"flat<float> SbnMaxSum"}
    assert items("sbn_step_flat<float, SbnLogSumExp>") == {"flat<float> SbnLogSumExp"}
    assert items("sbn_argmax_step") == {"argmax"}


def test_sum_product_names_map_to_the_items_they_always_had():
    assert items("sbn_step_batched<3, 0>") == {"batched N_IN=3", "batched CX=0"}
    assert items("sbn_step_batched<2, 8>") == {"batched N_IN=2", "batched CX=8"}
    assert items("sbn_step_flat<float>") == {"flat<float>"}
    assert items("sbn_step_flat<double>") == {"flat<double>"}
    assert items("sbn_step_batched_f64<5>") == {"batched_f64"}
    assert items("sbn_step_tiled<1, 1, 1, 0, 5, 2, 5, false, false>") == {
        "tiled (1,1,1,0)", "tiled T=5 CX=5", "tiled (1,1,1,0) T=5 CX=5"}
    assert items("sbn_marginal_step<double, 8>") == {"marginal<double,8>"}


def test_sum_product_and_policy_items_never_meet():
    sum_product = items("sbn_step_flat<float>", "sbn_step_flat<double>",
                        *[f"sbn_step_batched<{n}, {cx}>" for n in range(1, 9) for cx in (0, 1, 2, 3, 4, 5, 6, 8)])
    policy = items("sbn_step_flat<float, SbnMaxSum>", "sbn_step_flat<float, SbnLogSumExp>", "sbn_argmax_step",
                   *[f"sbn_step_batched<{n}, 0, {r}>" for n in range(1, 9) for r in ("SbnMaxSum", "SbnLogSumExp")])
    assert len(policy) == 19 and not sum_product & policy
