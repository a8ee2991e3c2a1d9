"""Hyper-parameter presets of the BASELINE.json configs as ARGs objects (values as shipped in the reference's
run/args/*.json; a user can equally pass those JSON files to run/main_from_args.py unchanged)."""
from openea_b200.modules.args.args_hander import ARGs

_COMMON = dict(training_data="../../datasets/", output="../../output/results/", dataset_division="721_5fold/1/",
               search_module="greedy", ordered=True, start_valid=100, eval_freq=10, stop_metric="hits1", csls=10,
               top_k=[1, 5, 10, 50], is_save=True, max_epoch=2000, batch_threads_num=2, test_threads_num=4)


def _args(**kw):
    d = dict(_COMMON)
    d.update(kw)
    return ARGs(d)


def mtranse(scale="15K", dim=100):
    return _args(embedding_module="MTransE", alignment_module="mapping", dim=dim, init="unit", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", learning_rate=0.01, optimizer="Adagrad",
                 batch_size=5000 if scale == "15K" else 20000, alpha=5, eval_metric="inner", eval_norm=True)


def bootea(scale="15K"):
    big = scale != "15K"
    return _args(embedding_module="BootEA", alignment_module="swapping", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss="limited", loss_norm="L2", learning_rate=0.01, optimizer="Adagrad",
                 batch_size=20000 if big else 5000, pos_margin=0.01, neg_margin=2.0, neg_margin_balance=0.2,
                 neg_sampling="truncated", neg_triple_num=10, truncated_epsilon=0.98 if big else 0.9, truncated_freq=10,
                 eval_metric="inner", eval_norm=False, sim_th=0.7, k=10, likelihood_slice=10,
                 sub_epoch=20 if big else 10, batch_threads_num=4 if big else 2, test_threads_num=12 if big else 4)


def aligne(scale="15K"):
    a = bootea(scale)
    a.embedding_module = "AlignE"
    return a


def transe(scale="15K"):
    return _args(embedding_module="TransE", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss="margin-based", loss_norm="L2", margin=1.5, learning_rate=0.01,
                 optimizer="Adagrad", batch_size=5000 if scale == "15K" else 20000, neg_sampling="uniform",
                 neg_triple_num=1, truncated_epsilon=0.9, truncated_freq=10, eval_metric="inner", eval_norm=True)


def gcn_align(scale="15K"):
    return _args(embedding_module="GCN_Align", alignment_module="mapping", dim=100, neg_sampling="uniform",
                 neg_triple_num=5, learning_rate=8, batch_size=5000, test_threads_num=3, eval_metric="manhattan",
                 eval_norm=False, support_number=1, se_dim=100, ae_dim=100, hidden1=100, gamma=3, early_stop=False,
                 dropout=0, test_method="sa", beta=0.9)


def alinet(scale="15K"):
    big = scale != "15K"
    return _args(embedding_module="AliNet", alignment_module="mapping", layer_dims=[500, 400, 300], init="xavier",
                 ent_l2_norm=True, rel_l2_norm=True, learning_rate=0.001, optimizer="Adam",
                 batch_size=20000 if big else 3000, neg_margin=1.5, neg_margin_balance=0.1, dropout=0.0,
                 neg_sampling="truncated", neg_triple_num=10, truncated_epsilon=0.995 if big else 0.98, truncated_freq=10,
                 start_valid=10, eval_metric="inner", eval_norm=False, is_save=False, min_rel_win=50 if not big else 15,
                 start_augment=2, rel_param=0.01, num_features_nonzero=0, sim_th=0.0, k=20)


def rdgcn(scale="15K"):
    big = scale != "15K"
    return _args(embedding_module="RDGCN", alignment_module="mapping", dim=300, neg_sampling="uniform",
                 neg_triple_num=10 if big else 125, learning_rate=0.001 if big else 0.002, batch_size=5000,
                 test_threads_num=3, start_valid=30, eval_metric="manhattan", eval_norm=False, gamma=1.0, dropout=0,
                 beta=0.3, alpha=0.1, synthetic_names=True)


def transh(scale="15K"):
    a = transe(scale)            # run/args/transh_args_*.json: TransE's settings, eval_norm false
    a.embedding_module, a.eval_norm = "TransH", False
    return a


def transd(scale="15K"):
    a = transh(scale)
    a.embedding_module = "TransD"
    return a


def transr(scale="15K"):
    """run/args/transr_args_15K.json (the reference ships the 15K configuration only)."""
    return _args(embedding_module="TransR", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", margin=1.5, loss="margin-based", neg_sampling="uniform",
                 neg_triple_num=1, learning_rate=0.01, optimizer="Adagrad", batch_size=5000, batch_threads_num=2,
                 test_threads_num=4, eval_metric="inner", eval_norm=False)


def proje(scale="15K"):
    """run/args/proje_args_15K.json and proje_args_100K.json."""
    small = scale == "15K"
    return _args(embedding_module="ProjE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                 rel_l2_norm=True, learning_rate=0.001, optimizer="Adam", batch_size=500 if small else 5000,
                 dnn_neg_nums=4096, batch_threads_num=2 if small else 3, test_threads_num=2 if small else 10,
                 start_valid=100 if small else 300, eval_metric="inner", eval_norm=True)


def conve(scale="15K"):
    """run/args/conve_args_15K.json and conve_args_100K.json: ProjE's settings plus the tower's."""
    a = proje(scale)
    a.embedding_module = "ConvE"
    a.output_keep_prob = 0.7
    a.filter_num = 32
    return a


def simple(scale="15K"):
    return _args(embedding_module="SimplE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                 rel_l2_norm=True, learning_rate=0.01, optimizer="Adagrad", batch_size=5000 if scale == "15K" else 20000,
                 neg_sampling="uniform", neg_triple_num=1, start_valid=10, test_threads_num=3, eval_metric="inner",
                 eval_norm=True)


def distmult(scale="15K"):
    a = simple(scale)            # the reference ships no distmult_args json; SimplE's settings fit its init()
    a.embedding_module = "DistMult"
    a.alpha = 5                  # DistMult.init builds the mapping graph unconditionally (distmult.py:27-30)
    return a


def rotate(scale="15K"):
    """run/args/rotate_args_*.json."""
    small = scale == "15K"
    return _args(embedding_module="RotatE", alignment_module="sharing", dim=100, init="uniform", ent_l2_norm=True,
                 rel_l2_norm=True, neg_sampling="uniform", neg_triple_num=10, gamma=12.0, learning_rate=0.1,
                 optimizer="Adam", batch_size=5000 if small else 20000, batch_threads_num=2 if small else 3,
                 test_threads_num=2 if small else 1, start_valid=200, eval_metric="inner", eval_norm=True)


def hole(scale="15K"):
    """run/args/hole_args_*.json."""
    small = scale == "15K"
    return _args(embedding_module="HolE", alignment_module="sharing", dim=100, init="xavier", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", margin=0.2, neg_sampling="uniform", neg_triple_num=1,
                 learning_rate=0.01, optimizer="Adagrad", batch_size=5000 if small else 20000,
                 batch_threads_num=2 if small else 3, test_threads_num=3 if small else 10, eval_metric="inner",
                 eval_norm=False)


def bootea_rotate(scale="15K"):
    """run/args/bootea_rotate_args_15K.json (the reference ships the 15K configuration only)."""
    return _args(embedding_module="BootEA_RotatE", alignment_module="swapping", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=False, gamma=12.0, learning_rate=0.01, optimizer="Adam", batch_size=5000, min_iter=40,
                 neg_sampling="uniform", neg_triple_num=10, truncated_epsilon=0.9, truncated_freq=10,
                 batch_threads_num=4, test_threads_num=4, start_valid=10, start_bp=5000, eval_metric="inner",
                 eval_norm=True, sim_th=0.75, k=10, sub_epoch=10, align_times=1)


def bootea_transh(scale="15K"):
    a = bootea(scale)
    a.embedding_module = "BootEA_TransH"
    return a


def iptranse(scale="15K"):
    """run/args/iptranse_args_*.json."""
    return _args(embedding_module="IPTransE", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", learning_rate=0.01, optimizer="Adagrad",
                 batch_size=5000 if scale == "15K" else 20000, margin=1.5, path_parm=0.1, neg_sampling="uniform",
                 neg_triple_num=1, eval_metric="inner", eval_norm=False, sim_th=0.7, bp_freq=100)


def sea(scale="15K"):
    """run/args/sea_args_*.json."""
    return _args(embedding_module="SEA", alignment_module="mapping", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", margin=1.5, loss="margin-based", alpha_1=2.5, alpha_2=0.25,
                 neg_sampling="uniform", neg_triple_num=1, learning_rate=0.01, optimizer="Adam",
                 batch_size=5000 if scale == "15K" else 20000, start_valid=10, eval_metric="inner", eval_norm=True)


def imuse(scale="15K"):
    """run/args/imuse_args_*.json."""
    return _args(embedding_module="IMUSE", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", margin=1.5, loss="margin-based", neg_sampling="uniform",
                 neg_triple_num=1, learning_rate=0.01, optimizer="SGD", batch_size=5000 if scale == "15K" else 20000,
                 start_valid=10, eval_metric="inner", eval_norm=True, sim_thresholds_ent=0.6, sim_thresholds_attr=0.6,
                 interactive_model_iter_num=1)


def attre(scale="15K"):
    """run/args/attre_args_*.json."""
    return _args(embedding_module="AttrE", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, attr_l2_norm=True, char_l2_norm=True, loss_norm="L2", margin=1.5, loss="margin-based",
                 neg_sampling="uniform", neg_triple_num=1, learning_rate=0.01, optimizer="SGD",
                 batch_size=5000 if scale == "15K" else 20000, eval_metric="inner", eval_norm=True, literal_len=5)


def attr2vec(scale="15K"):
    """JAPE's configuration (run/args/jape_args_*.json) with embedding_module = "Attr2Vec": the reference ships no
    configuration of its own for it."""
    a = jape(scale)
    a.embedding_module = "Attr2Vec"
    return a


def jape(scale="15K"):
    """run/args/jape_args_*.json."""
    return _args(embedding_module="JAPE", alignment_module="sharing", dim=100, init="normal", ent_l2_norm=True,
                 rel_l2_norm=True, loss_norm="L2", learning_rate=0.01, optimizer="Adagrad",
                 batch_size=5000 if scale == "15K" else 20000, attr_max_epoch=200, top_attr_threshold=0.9,
                 attr_sim_mat_threshold=0.95, attr_sim_mat_beta=0.001, neg_alpha=0.1, neg_sampling="uniform",
                 neg_triple_num=1, sub_mat_size=1000, eval_metric="inner", eval_norm=False)
