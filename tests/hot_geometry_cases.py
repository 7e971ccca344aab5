"""The dims at which tests/test_gpu_hot_geometry.py runs the hot-sign reduce (k_reduce_hot), one or two per geometry
class.  Plain data: tests/test_hot_geometry_classes.py checks, without a GPU, that every class the launcher can choose
(pb_hot_geometry over dims 1..4096, f16 and f32, one id per sample and ragged) holds one of them, so a launcher change
that adds a class fails there until the class gets a case here."""

SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
ALL = (SGD, ADAGRAD, ADAGRAD_VW, ADAM)
HOT_COLS = 512  # columns of a row per pass


def geometry_class(dim, g):
    """The class of a dim: what pb_hot_geometry returns, with the columns of a pass reduced to one or several passes
    and whether the last pass is short."""
    return (g["EPL"], g["CH"], g["PW"], g["vec"], g["vshift"], g["lean"], g["R1"], g["R"], g["S"], g["passes"] > 1,
            g["passes"] > 1 and dim % HOT_COLS != 0)


# one id per sample: (dim, f16, optimizers) at the smallest and largest dim of every class.  SGD everywhere, and one of
# Adagrad / vectorwise Adagrad / Adam in turn at each class's smallest dim; all four at a dim with dim % EPL != 0 (the
# optimizer step goes element by element) and at three and four chain warps.
ONE_ID_CASES = [
    # f32
    (1, False, ALL), (63, False, (SGD,)), (2, False, (SGD, ADAGRAD)), (62, False, (SGD,)),
    (4, False, (SGD, ADAGRAD_VW)), (8, False, (SGD, ADAM)), (16, False, (SGD, ADAGRAD)), (32, False, (SGD, ADAGRAD_VW)),
    (64, False, (SGD, ADAM)), (12, False, (SGD, ADAGRAD_VW)), (28, False, (SGD,)), (36, False, (SGD, ADAGRAD)),
    (40, False, (SGD, ADAM)), (44, False, (SGD, ADAGRAD_VW)), (48, False, (SGD,)), (52, False, (SGD, ADAGRAD)),
    (60, False, (SGD,)), (65, False, ALL), (71, False, (SGD,)), (66, False, (SGD, ADAM)), (70, False, (SGD,)),
    (68, False, (SGD, ADAM)), (84, False, (SGD,)), (73, False, ALL), (83, False, (SGD,)), (74, False, (SGD, ADAGRAD_VW)),
    (82, False, (SGD,)), (85, False, ALL), (99, False, (SGD,)), (86, False, (SGD, ADAGRAD)), (98, False, (SGD,)),
    (88, False, (SGD, ADAGRAD_VW)), (124, False, (SGD,)), (101, False, ALL), (127, False, (SGD,)),
    (102, False, (SGD, ADAM)), (126, False, (SGD,)), (128, False, (SGD, ADAGRAD)), (129, False, ALL),
    (167, False, (SGD,)), (132, False, (SGD, ADAM)), (252, False, (SGD,)), (169, False, ALL), (255, False, (SGD,)),
    (256, False, (SGD, ADAGRAD_VW)), (257, False, ALL), (384, False, (SGD,)), (385, False, ALL), (511, False, (SGD,)),
    (512, False, ALL), (513, False, ALL), (4095, False, (SGD,)), (516, False, ALL), (4092, False, (SGD,)),
    (1024, False, ALL), (4096, False, (SGD,)),
    # f16
    (1, True, ALL), (63, True, (SGD,)), (2, True, (SGD, ADAGRAD)), (62, True, (SGD,)), (8, True, (SGD, ADAGRAD_VW)),
    (16, True, (SGD, ADAM)), (32, True, (SGD, ADAGRAD)), (64, True, (SGD, ADAGRAD_VW)), (24, True, (SGD, ADAM)),
    (56, True, (SGD,)), (65, True, ALL), (71, True, (SGD,)), (66, True, (SGD, ADAGRAD)), (70, True, (SGD,)),
    (72, True, (SGD, ADAM)), (73, True, ALL), (83, True, (SGD,)), (74, True, (SGD, ADAM)), (84, True, (SGD,)),
    (80, True, (SGD, ADAGRAD_VW)), (85, True, ALL), (99, True, (SGD,)), (86, True, (SGD, ADAGRAD_VW)),
    (100, True, (SGD,)), (88, True, (SGD, ADAGRAD)), (96, True, (SGD,)), (101, True, ALL), (127, True, (SGD,)),
    (102, True, (SGD, ADAGRAD)), (126, True, (SGD,)), (104, True, (SGD, ADAM)), (120, True, (SGD,)),
    (128, True, (SGD, ADAGRAD_VW)), (129, True, ALL), (167, True, (SGD,)), (136, True, (SGD, ADAGRAD)),
    (168, True, (SGD,)), (169, True, ALL), (255, True, (SGD,)), (176, True, (SGD, ADAM)), (248, True, (SGD,)),
    (256, True, (SGD, ADAGRAD_VW)), (257, True, ALL), (383, True, (SGD,)), (264, True, ALL), (384, True, (SGD,)),
    (385, True, ALL), (511, True, (SGD,)), (392, True, ALL), (504, True, (SGD,)), (512, True, ALL), (513, True, ALL),
    (4095, True, (SGD,)), (520, True, ALL), (4088, True, (SGD,)), (1024, True, ALL), (4096, True, (SGD,)),
]

# several ids per sample, sqrt scaling and a loss scale: (dim, f16) for every class whose one-id form takes the
# producers' lean loop (ragged, the same dims take the general loop: classes of their own)
RAGGED_CASES = [(4, False), (8, False), (16, False), (32, False), (64, False), (128, False),
                (8, True), (16, True), (32, True), (64, True), (128, True), (256, True)]

# a slot of more than HOT_WIN samples with an item across the window boundary: (dim, f16), one per ring length S and
# producer mode (lean, 16-byte loads with a power-of-two or another vector count per row, element by element)
WINDOW_CASES = [(4, False), (256, False), (12, False), (1, False),
                (128, True), (512, True), (72, True), (65, False)]

# the sharded requester's instantiation (k_reduce_hot<..., SEND = true>): (dim, f16), one per (EPL, CH, 16-byte loads,
# S) and dtype, odd where the group has odd dims (the send area is then stored element by element)
SEND_CASES = [(2, False), (4, False), (65, False), (66, False), (68, False), (1, False), (129, False), (132, False),
              (257, False), (385, False),
              (2, True), (8, True), (65, True), (66, True), (72, True), (1, True), (129, True), (136, True),
              (257, True), (264, True), (385, True), (392, True)]
