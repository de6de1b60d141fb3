from .modules import ImageStem, MACModel, MACNetwork, OutputUnit, QuestionEncoder, answer_loss  # noqa: F401
