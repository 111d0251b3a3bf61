from omnisafe_b200.models.actor_critic import ConstraintActorCritic, ParamMap, param_layout  # noqa: F401
