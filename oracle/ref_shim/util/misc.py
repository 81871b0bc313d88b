"""Stand-in for the DINO package's util.misc: the detection backbone module imports only NestedTensor from it."""


class NestedTensor:
    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask
