"""Minimal attribute-namespace configuration (yacs is not available offline).

Only the keys the hot-path modules read, with the values of configs/pretrain/mq-glip-t.yaml and
maskrcnn_benchmark/config/defaults.py; a real yacs ``cfg`` object works in its place (same attribute paths).
"""
from types import SimpleNamespace as NS


def mq_glip_t_cfg(**over):
    cfg = NS(
        MODEL=NS(
            DEVICE="cuda",
            BACKBONE=NS(OUT_CHANNELS=256),
            SWINT=NS(EMBED_DIM=96, DEPTHS=(2, 2, 6, 2), NUM_HEADS=(3, 6, 12, 24), WINDOW_SIZE=7, MLP_RATIO=4,
                     OUT_CHANNELS=(96, 192, 384, 768)),
            LANGUAGE_BACKBONE=NS(LANG_DIM=768, MAX_QUERY_LEN=256, N_LAYERS=1, MODEL_TYPE="bert-base-uncased", PAD_MAX=True),
            GROUP_NORM=NS(NUM_GROUPS=16),
            RPN=NS(ASPECT_RATIOS=(1.0,), SCALES_PER_OCTAVE=1, ANCHOR_SIZES=(64, 128, 256, 512, 1024),
                   ANCHOR_STRIDE=(8, 16, 32, 64, 128), RETURN_FUSED_FEATURES=False),
            ROI_BOX_HEAD=NS(POOLER_RESOLUTION=7, POOLER_SCALES=(0.125, 0.0625, 0.03125, 0.015625, 0.0078125),
                            POOLER_SAMPLING_RATIO=0),
            ATSS=NS(INFERENCE_TH=0.05, PRE_NMS_TOP_N=1000, NMS_TH=0.6, DETECTIONS_PER_IMG=100, NUM_CLASSES=81),
            DYHEAD=NS(NUM_CLASSES=81, CHANNELS=256, NUM_CONVS=6, USE_GN=True, USE_DYRELU=True, USE_DFCONV=True,
                      USE_DYFUSE=True, PRIOR_PROB=0.01, LOG_SCALE=0.0, SCORE_AGG="MEAN",
                      FUSE_CONFIG=NS(EARLY_FUSE_ON=True, TYPE="MHA-B", JOINT_EMB_SIZE=256,
                                     USE_DOT_PRODUCT_TOKEN_LOSS=True, USE_FUSED_FEATURES_DOT_PRODUCT=True,
                                     USE_TOKEN_LOSS=False, USE_CONTRASTIVE_ALIGN_LOSS=False, MLM_LOSS=False,
                                     STABLE_SOFTMAX_2D=False, CLAMP_MIN_FOR_UNDERFLOW=True, CLAMP_MAX_FOR_OVERFLOW=True,
                                     CLAMP_BERTATTN_MIN_FOR_UNDERFLOW=True, CLAMP_BERTATTN_MAX_FOR_OVERFLOW=True,
                                     CLAMP_DOT_PRODUCT=True, SEPARATE_BIDIRECTIONAL=False,
                                     DO_LANG_PROJ_OUTSIDE_CHECKPOINT=False)),
        ),
        VISION_QUERY=NS(ENABLED=True, FIX_ATTN_GATE=-1.0, CONDITION_GATE=True, NONLINEAR_GATE=True, NO_CAT=True,
                        ADD_ADAPT_LAYER=False, RETURN_ATTN_GATE_VALUE=False, VISION_SCALE=1.0,
                        AUGMENT_IMAGE_WITH_QUERY=False, TEXT_DROPOUT=0.4, NEW_MASK_TOKEN=False, QUERY_FUSION=False,
                        SHARE_KV=False, NUM_QUERY_PER_CLASS=5, SELECT_FPN_LEVEL=True, QUERY_BANK_PATH="",
                        LEARNABLE_BANK=False, ADD_VISION_LAYER=False, PURE_TEXT_RATE=0.0, RANDOM_KSHOT=False,
                        EXPAND_RATIO=1.5, MAX_QUERY_NUMBER=5000, SIMILARITY_THRESHOLD=0.85,
                        MASK_DURING_INFERENCE=False,
                        # the test-time query update (engine/online_update.py), the values of config/defaults.py
                        SCORE_THRESHOLD=0.6, MAX_TEST_QUERY_NUMBER=100, NUM_TURNS=1, OFFLINE_WITH_ONLINE=False),
        # multi-scale / flip test-time augmentation (engine/bbox_aug.py), the values of config/defaults.py:856-867
        TEST=NS(MDETR_STYLE_AGGREGATE_CLASS_NUM=-1, USE_MULTISCALE=False,
                SCALES=(400, 500, 600, 640, 700, 900, 1000, 1100, 1200, 1300, 1400, 1800),
                RANGES=((96, 10000), (96, 10000), (64, 10000), (64, 10000), (64, 10000), (0, 10000), (0, 10000), (0, 256),
                        (0, 256), (0, 192), (0, 192), (0, 96)),
                MAX_SIZE=2500, FLIP=True, SPECIAL_NMS="none", TH=0.6, PRE_NMS_TOP_N=1000, NUM_CLASSES=81, SELECT_CLASSES=(),
                # images per test batch (the yaml's TEST block); read only by engine.batches.reference_test_batches
                IMS_PER_BATCH=8),
        # the test transform (engine/transforms.py): config/defaults.py:68-78 and the yaml's INPUT block
        INPUT=NS(PIXEL_MEAN=[103.530, 116.280, 123.675], PIXEL_STD=[57.375, 57.120, 58.395], MIN_SIZE_TEST=800, MAX_SIZE_TEST=1333,
                 FORMAT="", TO_BGR255=True),
        # ASPECT_RATIO_GROUPING: config/defaults.py:214; read only by engine.batches.reference_test_batches
        DATALOADER=NS(SIZE_DIVISIBILITY=32, ASPECT_RATIO_GROUPING=True),
    )
    for k, v in over.items():
        node = cfg
        parts = k.split(".")
        for p in parts[:-1]:
            node = getattr(node, p)
        setattr(node, parts[-1], v)
    return cfg


def mq_glip_l_cfg(**over):
    """configs/pretrain/mq-glip-l.yaml: Swin-L backbone (embed 192, depths 2/2/18/2, heads 6/12/24/48, window 12), 8 fusion
    layers; with the LVIS evaluation keys of configs/vision_query_5shot/lvis_minival.yaml (300 detections per prompt chunk,
    chunks of 40 classes, 3000 score columns in the reference's convert_grounding_to_od_logits_v2)."""
    base = {"MODEL.SWINT.EMBED_DIM": 192, "MODEL.SWINT.DEPTHS": (2, 2, 18, 2), "MODEL.SWINT.NUM_HEADS": (6, 12, 24, 48),
            "MODEL.SWINT.WINDOW_SIZE": 12, "MODEL.SWINT.OUT_CHANNELS": (192, 384, 768, 1536), "MODEL.DYHEAD.NUM_CONVS": 8,
            "MODEL.ATSS.DETECTIONS_PER_IMG": 300, "TEST.MDETR_STYLE_AGGREGATE_CLASS_NUM": 3000}
    base.update(over)
    cfg = mq_glip_t_cfg(**base)
    cfg.TEST.CHUNKED_EVALUATION = 40
    return cfg


def mq_groundingdino_t_cfg(**over):
    """configs/pretrain/mq-groundingdino-t.yaml + the GROUNDINGDINO block of maskrcnn_benchmark/config/defaults.py:944-1001
    (Swin-T with three outputs + one extra stride-2 level, 6 encoder / 6 decoder layers, 900 queries, two-stage "standard",
    text enhancer + fusion layers + text cross-attention, box threshold 0.05)."""
    base = {"INPUT.PIXEL_MEAN": [0.485, 0.456, 0.406], "INPUT.PIXEL_STD": [0.229, 0.224, 0.225], "INPUT.FORMAT": "rgb",
            "MODEL.ROI_BOX_HEAD.POOLER_SCALES": (0.125, 0.0625, 0.03125, 0.015625)}
    base.update(over)
    cfg = mq_glip_t_cfg(**{k: v for k, v in base.items() if not k.startswith("GROUNDINGDINO.")})
    cfg.GROUNDINGDINO = NS(
        enabled=True, modelname="groundingdino", backbone="swin_T_224_1k", position_embedding="sine", pe_temperatureH=20,
        pe_temperatureW=20, return_interm_indices=[1, 2, 3], enc_layers=6, dec_layers=6, pre_norm=False, dim_feedforward=2048,
        hidden_dim=256, dropout=0.0, nheads=8, num_queries=900, query_dim=4, num_patterns=0, num_feature_levels=4, enc_n_points=4,
        dec_n_points=4, two_stage_type="standard", two_stage_bbox_embed_share=False, two_stage_class_embed_share=False,
        transformer_activation="relu", dec_pred_bbox_embed_share=True, embed_init_tgt=True, max_text_len=256,
        text_encoder_type="bert-base-uncased", use_text_enhancer=True, use_fusion_layer=True, use_checkpoint=False,
        use_transformer_ckpt=False, use_text_cross_attention=True, text_dropout=0.0, fusion_dropout=0.0, fusion_droppath=0.1,
        sub_sentence_present=True, box_threshold=0.05, focal_alpha=0.25, loss_ce_coef=2.0, loss_bbox_coef=5.0, loss_giou_coef=2.0,
        matcher=NS(matcher_type="HungarianMatcher", set_cost_class=1.0, set_cost_bbox=5.0, set_cost_giou=2.0, focal_alpha=0.25))
    for k, v in base.items():
        if k.startswith("GROUNDINGDINO."):
            setattr(cfg.GROUNDINGDINO, k.split(".", 1)[1], v)
    return cfg
