from .launcher import Launcher, SurrealDefaultLauncher, PipelinedEngine, ReplayEngine  # noqa: F401
