from .layers import FeedforwardBlock, GatedFeedforwardBlock, TransformerEncoderLayer, name_to_block, name_to_input
from .emulator import EmulatedDMoE, EmulatedFaultyDMoE, get_non_expert_params
