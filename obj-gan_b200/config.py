"""Configuration object with the same shape as the reference's global ``cfg``
(reference: image_generation/miscc/config.py:9-87).  Only the keys the hot path and the
training loop read are kept; values are the reference defaults except TEXT.WORDS_NUM, which BASELINE.json
fixes at 18 tokens, and TEST.USE_TF, which defaults to 0 here (the reference's 1 selects its TensorFlow Inception
path, which this library does not implement; evaluator.condGANEvaluator refuses it)."""


class AttrDict(dict):
    """dict with attribute access (the reference uses easydict.EasyDict)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def default_cfg():
    c = AttrDict()
    c.GPU_IDS = "0"
    c.DATA_DIR = ""        # the dataset root; the snapshot PNGs' caption font is read below it (snapshots.py)
    c.CUDA = True
    c.RNN_TYPE = "LSTM"    # the text encoder's recurrent cell; RNN_ENCODER implements the LSTM only
    c.TREE = AttrDict(BRANCH_NUM=3, BASE_SIZE=64)
    c.TRAIN = AttrDict(
        BATCH_SIZE=16, DISCRIMINATOR_LR=2e-4, GENERATOR_LR=2e-4, BUATTN_NORM=True,
        # the training loop (trainer.condGANTrainer): epochs, snapshot / log intervals, the pretrained DAMSM text
        # encoder (the image encoder is the same path with text_encoder -> image_encoder) and a generator to resume
        MAX_EPOCH=60, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=100, DISPLAY_INTERVAL=500, FLAG=True,
        NET_E="/pretrained/text_encoder100.pth", NET_G="",
        SMOOTH=AttrDict(GAMMA1=4.0, GAMMA2=5.0, GAMMA3=10.0, DAMSM_LAMBDA=100.0,
                        TXT_LAMBDA=0.1, SHP_LAMBDA=1.0, OBJ_LAMBDA=0.1, UNCOND_LAMBDA=1.0))
    # the evaluator (evaluator.condGANEvaluator, ref: miscc/config.py:49-60): 0 ground-truth boxes and masks, 1
    # ground-truth boxes and generated masks, 2 generated boxes and masks; TEST_IMG_NUM counts batches, as there
    c.TEST = AttrDict(USE_GT_BOX_SEG=2, NET_SHP_G="/pretrained/shape_ckpt/shape_gen.pth", SAVE_OPTIONS="IMAGE",
                      FID_DIMS=2048, USE_TF=0, TEST_IMG_NUM=1000000, RP_POOL_SIZE=100, SAMPLE_VAL=False)
    c.GAN = AttrDict(DF_DIM=96, GF_DIM=48, Z_DIM=100, CONDITION_DIM=100, R_NUM=1,
                     LOCAL_R_NUM=3, GLB_R_NUM=7, LAYER_D_NUM=4)
    c.TEXT = AttrDict(CAPTIONS_PER_IMAGE=5, EMBEDDING_DIM=256, GLOVE_EMBEDDING_DIM=50,
                      WORDS_NUM=18)
    c.ROI = AttrDict(BOXES_NUM=10, BOXES_DIM=6, FM_SIZE=16, ROI_MIN_SIZE=10,
                     BOX_WORDS_NUM=1, ROI_BASE_SIZE=5, ROI_SIZE_THRS=16.0)
    return c


cfg = default_cfg()
