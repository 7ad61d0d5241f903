from ._encoders import OneHotEncoder
from .data import MinMaxScaler, QuantileTransformer, RobustScaler, StandardScaler
from .label import LabelEncoder

__all__ = ["StandardScaler", "MinMaxScaler", "RobustScaler", "QuantileTransformer", "LabelEncoder", "OneHotEncoder"]
